"""Conformance of the wgmma attention kernel (csrc/attention_wgmma.cu) through sr_test_attention_wgmma, against the
float64 reference of oracle/attn_oracle.py.

* Every output element lies within the oracle's bound, on every input family of attn_oracle.make_qkv (random,
  position-coded V, needles at the mask edges, an attention sink, a late-rising max, exact ties across blocks, uniform
  scores, large magnitudes), for packs whose lengths sit around every 64-row edge at unaligned offsets, 1 / 12 / 16
  heads, the MiniLM layout (dims 32-63 zero: those output columns exactly 0), the 256 x 512 headline pack, single
  sequences of 4 k - 32 k tokens (global attention at 16 k and 32 k on 1024+ sampled rows), windows 1 - 128 and >= len - 1,
  and key lengths 1, 63, 64, 65, len - 1, len in packs padded to 32 / 128 / 256 / 512.
* Bitwise: a sequence alone = inside a pack, other heads' inputs do not matter, kv_lens = len = no kv_lens, kv_lens > len
  = len, a larger max_len changes nothing, two runs agree, a length-1 sequence returns its V row.
* qkv rows past the pack are NaN and output rows past it hold sentinel bits that must survive; every row of the pack is
  written (the output starts as NaN).  Refused launches leave the output untouched.

Run with -s to see the largest |err| / bound per dominant error source."""
import numpy as np
import pytest
import torch

from oracle import attn_oracle as ao

pytestmark = pytest.mark.gpu

DEV = "cuda"
PAD_ROWS = 7
SENTINEL = 0x7E5A                      # an fp16 NaN payload no kernel writes
PACK = [5, 1, 2, 63, 64, 65, 127, 128, 129, 191, 192, 193, 3]
WINDOWS = [0, 1, 17, 63, 64, 65, 127, 128, 192]       # 192 = the longest length - 1: global
_STATS = {"ratio": {}, "tau": 0.0, "elements": 0}


@pytest.fixture(scope="module")
def lib(srlib, cuda):
    return srlib.hooks()


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if _STATS["ratio"]:
        print(f"\nattention: {_STATS['elements']} elements checked; largest |err| beyond eps per unit of coef "
              f"(TAU = {ao.TAU:.3e} must cover it): {_STATS['tau']:.3e}")
        print("largest |err| / bound where each source is the largest term of the bound:")
        for k in ao.SOURCES:
            if k in _STATS["ratio"]:
                print(f"  {k:9s} {_STATS['ratio'][k]:.3e}")


def _cu(lens):
    return [0] + np.cumsum(lens).tolist()


def _buffers(qkv, T, H):
    """qkv with NaN rows past T; output NaN below T and sentinel rows past it"""
    q = torch.full((T + PAD_ROWS, qkv.shape[1]), float("nan"), device=DEV, dtype=torch.float16)
    q[:T] = qkv
    out = torch.full((T + PAD_ROWS, H), float("nan"), device=DEV, dtype=torch.float16)
    out.view(torch.int16)[T:] = SENTINEL
    return q, out


def run(lib, qkv, cu, nH, window=0, kv_lens=None, max_len=None, head_dim=64, out=None):
    T = int(cu[-1])
    if out is None:
        qkv, out = _buffers(qkv, T, nH * 64)
    cu_d = torch.tensor(cu, dtype=torch.int32, device=DEV)
    kv_d = torch.tensor(kv_lens, dtype=torch.int32, device=DEV) if kv_lens is not None else None
    lens = [cu[i + 1] - cu[i] for i in range(len(cu) - 1)]
    ml = max(lens) if max_len is None else max_len
    rc = lib.sr_test_attention_wgmma(qkv.data_ptr(), out.data_ptr(), cu_d.data_ptr(), len(lens), ml, nH, head_dim, window,
                                     kv_d.data_ptr() if kv_d is not None else None)
    torch.cuda.synchronize()
    return rc, out


def check(name, got, ref):
    g = got.double()
    assert torch.isfinite(g).all(), f"{name}: an output row was not written (NaN left)"
    err = (g - ref.value).abs()
    bound = ref.bound()
    r = err / bound
    ratio = float(r.max())
    _STATS["elements"] += r.numel()
    _STATS["tau"] = max(_STATS["tau"], ref.tau_needed(got))
    terms = torch.stack([ref.terms[k] for k in ao.SOURCES])
    dom = terms.argmax(0)
    del terms
    for i, k in enumerate(ao.SOURCES):
        sel = r[dom == i]
        if sel.numel():
            _STATS["ratio"][k] = max(_STATS["ratio"].get(k, 0.0), float(sel.max()))
    if ratio > 1.0:
        i = int(r.argmax())
        raise AssertionError(f"{name}: |err| / bound = {ratio:.3g} at flat index {i} (row {i // g.shape[1]}, col "
                             f"{i % g.shape[1]}): got {g.flatten()[i].item()!r}, ref {ref.value.flatten()[i].item()!r}, "
                             f"bound {bound.flatten()[i].item():.3g}")


def _sentinels_kept(out, T):
    assert bool((out.view(torch.int16)[T:] == SENTINEL).all()), "an output row past the pack was written"


def _case(lib, name, family, lens, nH, window=0, kv=None, sel=None, seed=0, used=64):
    cu = _cu(lens)
    T = cu[-1]
    qkv = ao.make_qkv(family, cu, nH, window, kv, seed=seed, device=DEV, head_dim_used=used)
    rc, out = run(lib, qkv, cu, nH, window, kv)
    assert rc == 0
    _sentinels_kept(out, T)
    ref = ao.attention(qkv, cu, nH, window, kv, sel=sel)
    got = out[:T] if sel is None else out[sel]
    check(name, got, ref)
    return qkv, out[:T]


# ---- every family over the 64-row edges --------------------------------------------------------------------------------
FAMILY_CASES = [(w, 12) for w in WINDOWS] + [(w, h) for w in (0, 64) for h in (1, 16)]


@pytest.mark.parametrize("family", ao.FAMILIES)
@pytest.mark.parametrize("window,nH", FAMILY_CASES)
def test_families_around_the_row_edges(lib, family, window, nH):
    _case(lib, f"{family}/w{window}/h{nH}", family, PACK, nH, window, seed=window * 31 + nH)


@pytest.mark.parametrize("window", [0, 17, 64])
@pytest.mark.parametrize("lens", [[1, 2, 63, 64, 65], [129, 130, 700, 31], [128, 256, 127, 257, 5], [512], [2048]])
def test_mixed_packs(lib, lens, window):
    _case(lib, f"mixed{len(lens)}x{max(lens)}/w{window}", "random", lens, 12, window, seed=sum(lens) + window)


@pytest.mark.parametrize("window", [0, 64])
def test_minilm_layout(lib, window):
    """12 heads of 32 zero-padded to 64: the padded output columns are exactly 0"""
    _, out = _case(lib, f"minilm/w{window}", "random", PACK, 12, window, seed=5, used=32)
    assert bool((out.view(-1, 12, 64)[..., 32:].view(torch.int16) == 0).all())


@pytest.mark.parametrize("window", [0, 64])
def test_headline_pack(lib, window):
    _case(lib, f"headline/w{window}", "random", [512] * 256, 12, window, seed=6)


# ---- long single sequences -----------------------------------------------------------------------------------------
def _sampled_rows(L, n=1024, seed=0):
    g = torch.Generator().manual_seed(seed)
    tiles = (L + 63) // 64
    edges = [0, 63, (tiles // 2) * 64, (tiles // 2) * 64 + 63, (tiles - 1) * 64, L - 1]
    rows = torch.randperm(L, generator=g)[:n].tolist()
    return torch.tensor(sorted(set(rows + edges)), device=DEV)


@pytest.mark.parametrize("family", ["random", "position", "sink", "late"])
@pytest.mark.parametrize("window", [0, 64])
@pytest.mark.parametrize("L", [4096, 8192, 16384, 32768])
def test_long_sequence(lib, L, window, family):
    sel = _sampled_rows(L, seed=L) if (window == 0 and L >= 16384) else None
    _case(lib, f"long{L}/{family}/w{window}", family, [L], 1, window, sel=sel, seed=L + window)


# ---- key lengths (fixed-padding BERT) --------------------------------------------------------------------------------
@pytest.mark.parametrize("family", ["random", "needle"])
@pytest.mark.parametrize("L", [32, 128, 256, 512])
def test_kv_lens(lib, L, family):
    kvs = [1, 63, 64, 65, L - 1, L]
    _case(lib, f"kv{L}/{family}", family, [L] * len(kvs), 12, 0, kv=kvs, seed=L)


@pytest.mark.parametrize("L", [32, 128, 512])
def test_kv_lens_at_or_past_len_is_no_mask(lib, L):
    lens = [L, L - 1, 3, L]
    cu = _cu(lens)
    qkv = ao.make_qkv("random", cu, 12, seed=9, device=DEV)
    _, plain = run(lib, qkv, cu, 12)
    for kv in (lens, [x + 1 for x in lens], [x + 1000 for x in lens], [2 ** 31 - 1] * len(lens)):
        _, got = run(lib, qkv, cu, 12, 0, kv)
        assert torch.equal(got.view(torch.int16), plain.view(torch.int16)), kv


# ---- bitwise invariants -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("window", [0, 64])
def test_alone_equals_packed(lib, window):
    cu = _cu(PACK)
    qkv = ao.make_qkv("random", cu, 12, seed=11, device=DEV)
    _, packed = run(lib, qkv, cu, 12, window)
    for b, L in enumerate(PACK):
        _, alone = run(lib, qkv[cu[b]:cu[b + 1]].contiguous(), [0, L], 12, window)
        assert torch.equal(alone[:L].view(torch.int16), packed[cu[b]:cu[b + 1]].view(torch.int16)), (b, L)


@pytest.mark.parametrize("window", [0, 64])
def test_heads_are_independent(lib, window):
    cu = _cu(PACK)
    qkv = ao.make_qkv("random", cu, 16, seed=12, device=DEV)
    _, base = run(lib, qkv, cu, 16, window)
    other = ao.make_qkv("large", cu, 16, seed=13, device=DEV).view(-1, 3, 16, 64)
    mixed = other.clone()
    mixed[:, :, 5] = qkv.view(-1, 3, 16, 64)[:, :, 5]
    _, got = run(lib, mixed.view(-1, 3 * 16 * 64).contiguous(), cu, 16, window)
    h = slice(5 * 64, 6 * 64)
    assert torch.equal(got[:cu[-1], h].view(torch.int16), base[:cu[-1], h].view(torch.int16))


@pytest.mark.parametrize("window", [0, 64])
def test_max_len_and_repeat_change_nothing(lib, window):
    cu = _cu(PACK)
    qkv = ao.make_qkv("sink", cu, 12, seed=14, device=DEV)
    _, a = run(lib, qkv, cu, 12, window)
    _, b = run(lib, qkv, cu, 12, window)
    _, c = run(lib, qkv, cu, 12, window, max_len=max(PACK) + 200)
    assert torch.equal(a.view(torch.int16), b.view(torch.int16))
    assert torch.equal(a.view(torch.int16), c.view(torch.int16))


@pytest.mark.parametrize("window", [0, 1, 64])
def test_length_one_returns_its_v_row(lib, window):
    lens = [1, 5, 1, 1]
    cu = _cu(lens)
    qkv = ao.make_qkv("large", cu, 12, seed=15, device=DEV)
    _, out = run(lib, qkv, cu, 12, window, kv_lens=[1, 5, 7, 1] if window == 0 else None)
    v = qkv.view(-1, 3, 12 * 64)[:, 2]
    for b in (0, 2, 3):
        assert torch.equal(out[cu[b]].view(torch.int16), v[cu[b]].view(torch.int16)), b


# ---- refusals -----------------------------------------------------------------------------------------------------------
def test_refusals_leave_the_output_alone(lib):
    cu = _cu([70, 10])
    T = cu[-1]
    qkv = ao.make_qkv("random", cu, 12, seed=16, device=DEV)
    for kw in ({"window": 64, "kv_lens": [70, 10]}, {"head_dim": 32}, {"head_dim": 128}):
        q, out = _buffers(qkv, T, 12 * 64)
        out.view(torch.int16)[:] = SENTINEL
        rc, out = run(lib, q, cu, 12, out=out, **kw)
        assert rc != 0, kw
        assert bool((out.view(torch.int16) == SENTINEL).all()), kw
