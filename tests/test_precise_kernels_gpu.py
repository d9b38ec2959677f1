"""Conformance of the precise path's kernels (csrc/precise.cu) through their hooks (sr_test_precise_split / _rope /
_geglu / _attention) and of its triple-depth GEMM through sr_test_gemm_desc, element by element against the float64
references and bounds of oracle/precise_oracle.py and gemm_oracle.gemm(split=True).

  * Split: every width the loader accepts (H 384 / 768 / 1024, I 320 / 1088 / 1152 / 2624 / 4096), T = 1, 7, 8, 9, 255
    and 131 072, values at +-65 504, 2^-14 and below it (fp16-subnormal hi and lo), fp32 subnormals, 0 and -0: hi and lo
    bitwise fp16_rn(v) and fp16_rn(v - hi), the third part bitwise hi.  The LayerNorm variant: hi + lo within the bound
    of float64 LN, on rows of tiny variance, at eps 1e-5 and 1e-6.
  * RoPE on 1 / 12 / 16 heads, packs whose positions restart per sequence, positions up to 32 767, T up to 131 072.
  * GeGLU at every I above, a over [-10, 10] on a dense grid (the cancelling tail a <~ -4 included), T x I not a
    multiple of 256.
  * Attention on every family of precise_oracle.make_qkv (attn_oracle's and constant V under uniform scores), windows
    1, 31, 32, 33, 64, 128 and >= len - 1 over a pack of lengths 1 ... 129 at unaligned offsets, 1 / 12 / 16 heads,
    global attention over 8 192 and 32 768 keys on >= 1 024 sampled rows; bitwise: alone = in a pack, a length-1
    sequence returns its V row, a repeat call and a larger max_len change nothing.
  * Packs of 65 535, 65 536 and 70 000 one- and two-token sequences through both attention hooks (gridDim.z holds at
    most 65 535), and 70 000 sequences through sr_forward_dev on both paths, bitwise the same rows as two calls.
  * The triple-depth GEMM at every (N, K') encoder_forward_precise launches at those geometries, K' up to 12 288,
    M = 1, 127, 128, 129 and 17 370, EPI_RESID plain and in place.
  * The precise forward of a small ModernBERT and a small BERT model on a caller's stream (sr_model_set_stream): no
    device-bytes change from set_precise, launch counts exact at 1 and 2 attention slices per layer, and a CUDA graph
    capture of sr_forward_dev whose replay is bitwise the eager call.
Outputs start as NaN and rows past the launch hold sentinels that must survive.  Run with -s for the worst error / bound
of each kernel and where it occurs."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from oracle import attn_oracle as ao, encoder_oracle as eo, gemm_oracle as go, hidden_oracle as ho, precise_oracle as po
from oracle import synth

pytestmark = pytest.mark.gpu

DEV = "cuda"
WIDTHS = [384, 768, 1024, 320, 1088, 1152, 2624, 4096]
PACK = [1, 63, 64, 65, 127, 128, 129, 5]
_WORST = {}


@pytest.fixture(scope="module")
def lib(srlib, cuda):
    return srlib.hooks()


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for k, (r, where) in sorted(_WORST.items()):
        print(f"\nprecise {k}: worst |err| / bound {r:.3e} at {where}")


def _note(kernel, ratio, where):
    if ratio >= _WORST.get(kernel, (-1.0, ""))[0]:
        _WORST[kernel] = (ratio, where)


def _within(kernel, where, got, value, bound):
    g = got.double()
    assert bool(torch.isfinite(g).all()), f"{kernel} {where}: a non-finite output"
    r = (g - value).abs() / bound
    ratio = float(r.max()) if r.numel() else 0.0
    _note(kernel, ratio, where)
    if ratio > 1.0:
        i = int(r.argmax())
        raise AssertionError(f"{kernel} {where}: |err| / bound = {ratio:.3g} at flat {i}: got {g.flatten()[i].item()!r}, "
                             f"ref {value.flatten()[i].item()!r}, bound {bound.flatten()[i].item():.3g}")


def _cu(lens):
    return [0] + np.cumsum(lens).tolist()


# ---- split ---------------------------------------------------------------------------------------------------------
SPECIALS = [65504.0, -65504.0, 2.0 ** -14, -(2.0 ** -14), 0.75 * 2.0 ** -14, 2.0 ** -20 + 2.0 ** -31, 2.0 ** -24,
            2.0 ** -26, 1e-40, -1e-40, 0.0, -0.0, 1.0 + 2.0 ** -20, 0.1, -3.0e-3, 2.0 ** -5 + 2.0 ** -29]


def _split_rows(T, H, seed, tiny=False):
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(T, H, generator=g, device=DEV) * torch.exp(2 * torch.randn(T, 1, generator=g, device=DEV))
    sp = torch.tensor(SPECIALS, device=DEV)
    x[0, :len(SPECIALS)] = sp[:min(len(SPECIALS), H)]
    if T > 3:
        x[1] = 2.0 ** -10 * torch.randn(H, generator=g, device=DEV)           # lo in the fp16 subnormals
    if tiny:                                                                 # LN rows of tiny variance
        x[T // 2] = 1000.0 + 1e-3 * torch.randn(H, generator=g, device=DEV)
        x[-1] = 7.0
        x[-1, ::7] = 7.0 + 2.0 ** -21
    return x.contiguous()


def _run_split(lib, x, gamma, eps):
    T, H = x.shape
    out = torch.full((T + 2, 3 * H), float("nan"), device=DEV, dtype=torch.float16)
    out.view(torch.int16)[T:] = 0x7E5A
    assert lib.sr_test_precise_split(x.data_ptr(), T, H, gamma.data_ptr() if gamma is not None else None, eps,
                                     out.data_ptr()) == 0
    torch.cuda.synchronize()
    assert bool((out.view(torch.int16)[T:] == 0x7E5A).all()), "a row past T was written"
    return out[:T].view(T, 3, H)


@pytest.mark.parametrize("H", WIDTHS)
@pytest.mark.parametrize("T", [1, 7, 8, 9, 255])
def test_split_plain_is_bitwise(lib, H, T):
    x = _split_rows(T, H, seed=H + T)
    out = _run_split(lib, x, None, 0.0)
    hi, lo = po.split_halves(x.cpu().numpy())
    got = out.cpu().numpy()
    assert np.array_equal(got[:, 0].view(np.int16), hi.view(np.int16))
    assert np.array_equal(got[:, 1].view(np.int16), lo.view(np.int16))
    assert np.array_equal(got[:, 2].view(np.int16), hi.view(np.int16))


def _check_split_ln(lib, x, eps, where):
    H = x.shape[1]
    g = torch.Generator(device=DEV).manual_seed(H)
    gamma = torch.exp(torch.empty(H, device=DEV).uniform_(math.log(0.05), math.log(8.0), generator=g))
    out = _run_split(lib, x, gamma, eps)
    assert torch.equal(out[:, 0].view(torch.int16), out[:, 2].view(torch.int16))
    ref = po.split_ln(x, gamma, eps)
    _within("split+LN", where, out[:, 0].double() + out[:, 1].double(), ref.value, ref.bound)


@pytest.mark.parametrize("eps", [1e-5, 1e-6])
@pytest.mark.parametrize("H", WIDTHS)
@pytest.mark.parametrize("T", [1, 7, 9, 255])
def test_split_layernorm_within_bound(lib, H, T, eps):
    _check_split_ln(lib, _split_rows(T, H, seed=3 * H + T, tiny=True), eps, f"H {H} T {T} eps {eps}")


@pytest.mark.parametrize("ln", [False, True])
def test_split_131072_rows(lib, ln):
    x = _split_rows(131072, 768, seed=5, tiny=True)
    if ln:
        _check_split_ln(lib, x, 1e-5, "H 768 T 131072")
    else:
        got = _run_split(lib, x, None, 0.0).cpu().numpy()
        hi, lo = po.split_halves(x.cpu().numpy())
        assert np.array_equal(got[:, 0].view(np.int16), hi.view(np.int16))
        assert np.array_equal(got[:, 1].view(np.int16), lo.view(np.int16))


# ---- RoPE ----------------------------------------------------------------------------------------------------------
def _positions(cu):
    return torch.cat([torch.arange(cu[b + 1] - cu[b]) for b in range(len(cu) - 1)]).to(torch.int32)


@pytest.mark.parametrize("heads,lens,offset", [
    (1, [1, 63, 64, 65, 300], 0), (12, PACK, 0), (16, [129, 7, 1000], 0), (12, [2048], 30719), (1, [32768], 0),
    (12, [512] * 256, 0),
])
def test_rope_within_bound(lib, heads, lens, offset):
    cu = _cu(lens)
    T = cu[-1]
    pos = (_positions(cu) + offset).to(DEV)
    cos_t, sin_t = (t.to(DEV) for t in eo.rope_tables(64, 160000.0, int(pos.max()) + 1))
    g = torch.Generator(device=DEV).manual_seed(heads * 7 + T)
    qkv = 3 * torch.randn(T, 3 * heads * 64, generator=g, device=DEV)
    ref = po.rope(qkv, pos, heads, cos_t, sin_t)
    buf = qkv.clone()
    assert lib.sr_test_precise_rope(buf.data_ptr(), pos.data_ptr(), T, heads, cos_t.data_ptr(), sin_t.data_ptr()) == 0
    torch.cuda.synchronize()
    H = heads * 64
    assert torch.equal(buf[:, 2 * H:].view(torch.int32), qkv[:, 2 * H:].view(torch.int32)), "v third changed"
    _within("rope", f"heads {heads} T {T} positions to {int(pos.max())}", buf[:, :2 * H], ref.value[:, :2 * H],
            ref.bound[:, :2 * H] + 2.0 ** -140)


# ---- GeGLU ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("I", WIDTHS)
@pytest.mark.parametrize("T", [7, 33])
def test_geglu_within_bound(lib, I, T):
    g = torch.Generator(device=DEV).manual_seed(I + T)
    a = torch.linspace(-10.0, 10.0, T * I, device=DEV).view(T, I)
    b = torch.randn(T, I, generator=g, device=DEV) * 2
    ab = torch.cat([a, b], 1).contiguous()
    out = torch.full((T * I + 300,), float("nan"), device=DEV)
    out[T * I:] = 12345.0
    assert lib.sr_test_precise_geglu(ab.data_ptr(), T, I, out.data_ptr()) == 0
    torch.cuda.synchronize()
    assert bool((out[T * I:] == 12345.0).all()), "an element past T x I was written"
    ref = po.geglu(ab, I)
    _within("geglu", f"I {I} T {T}", out[:T * I].view(T, I), ref.value, ref.bound)


# ---- attention -----------------------------------------------------------------------------------------------------
def run_attn(lib, qkv, cu, heads, window=0, max_len=None):
    T = int(cu[-1])
    out = torch.full((T + 3, heads * 64), float("nan"), device=DEV)
    out[T:] = 4242.0
    cu_d = torch.tensor(cu, dtype=torch.int32, device=DEV)
    lens = [cu[i + 1] - cu[i] for i in range(len(cu) - 1)]
    ml = max(lens) if max_len is None else max_len
    assert lib.sr_test_precise_attention(qkv.data_ptr(), out.data_ptr(), cu_d.data_ptr(), len(lens), ml, heads, window) == 0
    torch.cuda.synchronize()
    assert bool((out[T:] == 4242.0).all()), "a row past the pack was written"
    return out[:T]


def _attn_case(lib, family, lens, heads, window, sel=None, seed=0):
    cu = _cu(lens)
    qkv = po.make_qkv(family, cu, heads, window, seed=seed, device=DEV)
    out = run_attn(lib, qkv, cu, heads, window)
    ref = po.attention(qkv, cu, heads, window, sel=sel)
    got = out if sel is None else out[sel]
    _within("attention", f"{family} lens {lens if len(lens) < 10 else len(lens)} heads {heads} window {window}", got,
            ref.value, ref.bound)
    if family == "constant":                      # every output element is its column's constant
        c = po.constant_columns().double().to(DEV).repeat(heads)
        _within("attention", f"constant/value heads {heads} window {window}", got, c.expand_as(got), ref.bound)
    return qkv, out


@pytest.mark.parametrize("family", po.FAMILIES)
@pytest.mark.parametrize("window,heads", [(w, 12) for w in (0, 1, 31, 32, 33, 64, 128, 128 + 1)] + [(0, 1), (64, 16)])
def test_attention_families(lib, family, window, heads):
    _attn_case(lib, family, PACK, heads, window, seed=window * 13 + heads)


def _sampled(L, n=1024, seed=0):
    g = torch.Generator().manual_seed(seed)
    edges = [0, 31, 32, 63, 64, L // 2, L - 65, L - 64, L - 1]
    return torch.tensor(sorted(set(torch.randperm(L, generator=g)[:n].tolist() + edges)), device=DEV)


@pytest.mark.parametrize("family,heads", [("random", 2), ("constant", 1), ("sink", 1), ("late", 2)])
@pytest.mark.parametrize("L", [8192, 32768])
def test_attention_global_long(lib, L, family, heads):
    _attn_case(lib, family, [L], heads, 0, sel=_sampled(L, seed=L), seed=L)


def test_attention_alone_equals_packed_and_repeats(lib):
    cu = _cu(PACK)
    for window in (0, 33):
        qkv = po.make_qkv("random", cu, 12, seed=21, device=DEV)
        packed = run_attn(lib, qkv, cu, 12, window)
        again = run_attn(lib, qkv, cu, 12, window, max_len=max(PACK) + 200)
        assert torch.equal(packed.view(torch.int32), again.view(torch.int32))
        assert torch.equal(packed.view(torch.int32), run_attn(lib, qkv, cu, 12, window).view(torch.int32))
        for b, L in enumerate(PACK):
            alone = run_attn(lib, qkv[cu[b]:cu[b + 1]].contiguous(), [0, L], 12, window)
            assert torch.equal(alone.view(torch.int32), packed[cu[b]:cu[b + 1]].view(torch.int32)), (window, b)


@pytest.mark.parametrize("window", [0, 1, 64])
def test_attention_length_one_returns_its_v_row(lib, window):
    lens = [1, 5, 1, 1]
    cu = _cu(lens)
    qkv = po.make_qkv("large", cu, 12, seed=22, device=DEV)
    out = run_attn(lib, qkv, cu, 12, window)
    v = qkv.view(-1, 3, 12 * 64)[:, 2]
    for b in (0, 2, 3):
        assert torch.equal(out[cu[b]].view(torch.int32), v[cu[b]].view(torch.int32)), b


# ---- more sequences than gridDim.z holds -----------------------------------------------------------------------------
def _subpack(qkv, cu, seqs):
    """the rows of sequences `seqs` as a pack of their own"""
    rows = torch.cat([torch.arange(cu[b], cu[b + 1]) for b in seqs]).to(qkv.device)
    return qkv[rows].contiguous(), _cu([cu[b + 1] - cu[b] for b in seqs]), rows


@pytest.mark.parametrize("B", [65535, 65536, 70000])
def test_attention_beyond_grid_z(lib, B):
    lens = [1 + (b % 3 == 1) for b in range(B)]
    cu = _cu(lens)
    check = sorted(set(list(range(8)) + list(range(65528, min(B, 65545))) + list(range(B - 8, B))))
    # V holds no zeros: a length-1 row is 0 + 1 * v, which turns -0 into +0
    nonzero = lambda x: torch.where(x == 0, torch.ones_like(x), x)
    # precise path: fp32
    qkv = nonzero(po.make_qkv("random", cu, 2, seed=B, device=DEV))
    out = run_attn(lib, qkv, cu, 2)
    one = torch.tensor([cu[b] for b in range(B) if lens[b] == 1], device=DEV)
    v = qkv.view(-1, 3, 128)[:, 2]
    assert torch.equal(out[one].view(torch.int32), v[one].view(torch.int32))
    sub, scu, rows = _subpack(qkv, cu, check)
    ref = po.attention(sub, scu, 2, 0)
    _within("attention", f"{B} sequences", out[rows], ref.value, ref.bound)
    # production path: the wgmma kernel, fp16
    q16 = nonzero(ao.make_qkv("random", cu, 2, seed=B, device=DEV))
    o16 = torch.full((cu[-1] + 1, 128), float("nan"), device=DEV, dtype=torch.float16)
    cu_d = torch.tensor(cu, dtype=torch.int32, device=DEV)
    assert lib.sr_test_attention_wgmma(q16.data_ptr(), o16.data_ptr(), cu_d.data_ptr(), B, 2, 2, 64, 0, None) == 0
    torch.cuda.synchronize()
    v16 = q16.view(-1, 3, 128)[:, 2]
    assert torch.equal(o16[one].view(torch.int16), v16[one].view(torch.int16))
    sub, scu, rows = _subpack(q16, cu, check)
    r16 = ao.attention(sub, scu, 2, 0)
    g = o16[rows].double()
    assert bool(((g - r16.value).abs() <= r16.bound()).all()), f"wgmma attention, {B} sequences"


@pytest.mark.parametrize("precise", [False, True])
def test_forward_beyond_grid_z_equals_two_calls(srlib, cuda, precise):
    from test_encoder_hidden_conformance_gpu import _forward, _load, _same
    cfg = ho.modernbert_config("small-384", 2)
    w = ho.modernbert_weights(cfg, "plain")
    rng = np.random.default_rng(7)
    seqs = synth.make_ids(rng, [1 + (b % 2) for b in range(70000)], cfg.vocab_size)
    with _load(srlib, cfg, w) as m:
        m.set_precise(precise)
        whole = _forward(srlib, m, seqs, 2)
        first = _forward(srlib, m, seqs[:65535], 2)
        second = _forward(srlib, m, seqs[65535:], 2)
        m.set_precise(False)
    assert _same(whole, torch.cat([first, second]))


# ---- the precise forward on a caller's stream ------------------------------------------------------------------------
def _small_model(arch):
    if arch == "modernbert":
        cfg = ho.modernbert_config("small-384", 2)
        return cfg, ho.modernbert_weights(cfg, "plain")
    cfg = eo.BertConfig(vocab_size=ho.VOCAB, hidden_size=384, num_hidden_layers=2, num_attention_heads=12,
                        intermediate_size=1536)
    return cfg, synth.make_bert_weights(cfg, 0, seed=31, with_pooler=False)


@pytest.mark.parametrize("lens", [PACK, [1] * 70000], ids=["pack", "70000-ones"])
@pytest.mark.parametrize("arch", ["modernbert", "bert"])
def test_forward_on_caller_stream_replays_as_a_graph(srlib, cuda, arch, lens):
    """sr_reserve, then set_precise(True), on a caller's stream: set_precise leaves device_bytes() unchanged, one eager
    forward counts exactly the kernels it launches (attention once per slice of at most 65 535 sequences), and the
    forward captures as a CUDA graph whose replay writes the eager call's hidden rows bitwise"""
    from test_encoder_hidden_conformance_gpu import _hidden, _load, _same
    cfg, w = _small_model(arch)
    L = srlib.lib()
    L.sr_launch_count.restype = C.c_longlong
    ids, cu = srlib.pack(synth.make_ids(np.random.default_rng(32), lens, cfg.vocab_size))
    T, B, max_len = len(ids), len(lens), max(lens)
    d_ids, d_cu = torch.from_numpy(ids).to(DEV), torch.from_numpy(cu).to(DEV)
    stream = torch.cuda.Stream()
    torch.cuda.synchronize()
    layers = cfg.num_hidden_layers
    slices = (B + 65534) // 65535
    # positions + embedding, then per layer 4 splits, 4 GEMMs, the attention slices and
    # ModernBERT: RoPE + GeGLU / BERT: GELU + 2 LayerNorms
    expected = 2 + layers * (8 + slices + (2 if arch == "modernbert" else 3))
    with _load(srlib, cfg, w) as m:
        h = m.handle
        assert L.sr_model_set_stream(h, C.c_void_p(stream.cuda_stream)) == 0
        assert L.sr_reserve(h, T, B, B) == 0
        loaded = m.device_bytes()
        m.set_precise(True)
        assert m.device_bytes() == loaded
        forward = lambda: L.sr_forward_dev(h, d_ids.data_ptr(), d_cu.data_ptr(), B, T, max_len, 0)
        with torch.cuda.stream(stream):
            n0 = L.sr_launch_count()
            assert forward() == 0
            assert L.sr_launch_count() - n0 == expected
        stream.synchronize()
        eager = _hidden(srlib, m, T)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=stream, capture_error_mode="thread_local"):
            assert forward() == 0

        class _Rows:
            __cuda_array_interface__ = {"data": (int(L.sr_dev_hidden(h)), False), "shape": (T, m.hidden),
                                        "typestr": "<f4", "version": 3}
        rows = torch.as_tensor(_Rows(), device=DEV)    # the model's hidden rows, not a copy
        with torch.cuda.stream(stream):
            rows.fill_(float("nan"))
            graph.replay()
        stream.synchronize()
        assert _same(rows.clone(), eager)
        assert L.sr_model_set_stream(h, None) == 0


# ---- the triple-depth GEMM -----------------------------------------------------------------------------------------
def _gemm_shapes():
    """(N, K) of every projection encoder_forward_precise launches at the loader's geometries"""
    shapes = set()
    for geo in ho.GEOMETRIES.values():
        H, I = geo["hidden_size"], geo["intermediate_size"]
        shapes |= {(3 * H, H), (H, H), (2 * I, H), (H, I)}
    return sorted(shapes)


def _gemm_case(M, N, K, in_place, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    a = torch.randn(M, K, generator=g, device=DEV)
    w = 0.02 * torch.randn(N, K, generator=g, device=DEV)
    a3, w3 = go.split3(a, w)
    rows = (M + 127) // 128 * 128
    A = torch.zeros(rows, 3 * K, dtype=torch.float16, device=DEV)
    A[:M] = a3
    out = torch.full((M, N), float("nan"), device=DEV)
    resid = None
    if in_place:
        resid = torch.randn(M, N, generator=g, device=DEV)
        out.copy_(resid)
    return a, w, A, w3, out, resid


@pytest.mark.parametrize("N,K", _gemm_shapes())
def test_triple_depth_gemm(lib, srlib, N, K):
    for M in (1, 127, 128, 129, 17370):
        for in_place in ((False, True) if M in (129, 17370) else (False,)):
            a, w, A, w3, out, resid = _gemm_case(M, N, K, in_place, seed=M + N + K)
            rc, _ = srlib.binding.run_gemm(m=M, n=N, k=3 * K, a=A, a_rows=A.shape[0], w=w3, out=out, ldo=N, epi=go.EPI_RESID,
                                   resid=out if in_place else 0, ldr=N)
            torch.cuda.synchronize()
            assert rc == 0
            ref = go.gemm(go.EPI_RESID, a, w, N, resid=resid, split=True)
            where = f"M {M} N {N} K' {3 * K}{' in place' if in_place else ''}"
            _note(f"gemm x3 (|err| - eps) / S' at K' {3 * K}", ref.tau_needed(out) * go.depth_scale(3 * K), where)
            _within("gemm x3", where, out, ref.value, ref.bound())
            del ref, a, w, A, w3, out
