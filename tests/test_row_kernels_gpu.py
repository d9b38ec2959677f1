"""Conformance of the row kernels of csrc/elementwise.cu (embeddings, LayerNorm rows, positions, cast, pooling, L2
normalisation, sequence and token heads) through their test hooks, against the float64 reference of
oracle/row_oracle.py.

* Every float output is within the derived bound of every element; every integer output (position, class,
  prediction) is exact, and so are the cast and the low half of the fp16 pair.
* Inputs are chosen so that each parameter moves the output by far more than the bound: rows of small variance (the
  LayerNorm eps shows), pre-activations in |x| in [1, 3] (tanh and erf GELU differ by ~1e-3), biases and type rows
  as large as the signal, rows of tiny norm (the L2 eps shows).
* Exact ties are built from duplicated classifier rows with equal biases, which give bit-identical logits.
* Output rows past the launch and refused launches must leave NaN sentinels in place.

Run with -s to see the largest |err| / bound per launcher."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import row_oracle as ro

pytestmark = pytest.mark.gpu

DEV = "cuda"
_RATIO = {}


@pytest.fixture(scope="module")
def lib(srlib, cuda):
    return srlib.hooks()


@pytest.fixture(scope="module")
def SeqW(srlib):
    return srlib.binding.SeqHeadWeights


@pytest.fixture(scope="module", autouse=True)
def _ratio_report():
    yield
    if _RATIO:
        print("\nlargest |err| / bound per launcher:")
        for k in sorted(_RATIO):
            print(f"  {k:22s} {_RATIO[k]:.3e}")


def _p(t):
    return None if t is None else t.data_ptr()


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _nan(*shape, dtype=torch.float32):
    return torch.full(shape, float("nan"), device=DEV, dtype=dtype)


def check(name, got, ref, mask=None):
    """every element of `got` within ref's bound (rows selected by `mask`)"""
    g = got.double()
    v, b = ref.value, ref.eps
    if mask is not None:
        g, v, b = g[mask], v[mask], b[mask]
    err = (g - v).abs()
    assert torch.isfinite(g).all(), f"{name}: non-finite output"
    r = torch.where(err == 0, torch.zeros_like(err), err / b)   # a zero bound (exact copy) demands a zero error
    ratio = float(r.max()) if r.numel() else 0.0
    _RATIO[name] = max(_RATIO.get(name, 0.0), ratio)
    if ratio > 1.0:
        i = int(r.argmax())
        raise AssertionError(f"{name}: |err| / bound = {ratio:.3g} at flat index {i}: got {g.flatten()[i].item()!r}, "
                             f"ref {v.flatten()[i].item()!r}, bound {b.flatten()[i].item():.3g}")


def _rows(T, H, g, mean=0.5, small_every=3):
    """rows with a per-row offset; every `small_every`-th row has a variance of ~1e-4, where eps 1e-5 shows"""
    x = torch.randn(T, H, device=DEV, generator=g)
    x[::small_every] *= 1e-2
    return (x + mean * torch.randn(T, 1, device=DEV, generator=g)).contiguous()


def _ids(T, vocab, g):
    ids = torch.randint(0, vocab, (T,), device=DEV, generator=g, dtype=torch.int32)
    edge = torch.tensor([0, vocab - 1, -1, vocab, 2 ** 31 - 1], device=DEV, dtype=torch.int32)
    n = min(T, len(edge))
    ids[:n] = edge[:n]
    if T > len(edge):
        ids[-n:] = edge[:n]
    return ids


# ---- embeddings -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("H", [384, 768, 1024])
@pytest.mark.parametrize("T", [1, 7, 8, 9, 1037, 65537])
def test_embed_ln_modernbert(lib, H, T):
    vocab, eps = 1000, 1e-5
    g = _gen(T * 7 + H)
    table = _rows(vocab, H, g)
    w = (1.0 + 0.5 * torch.randn(H, device=DEV, generator=g)).contiguous()
    ids = _ids(T, vocab, g)
    x, h = _nan(T + 8, H), _nan(T + 8, H, dtype=torch.float16)
    assert lib.sr_test_embed_ln_modernbert(_p(ids), T, H, vocab, _p(table), _p(w), eps, _p(x), _p(h), None) == 0
    torch.cuda.synchronize()
    ref = ro.embed_ln_modernbert(ids, table, w, eps)
    check("embed_ln_modernbert.x", x[:T], ref)
    check("embed_ln_modernbert.h", h[:T], ro.f16_out(ref))
    assert x[T:].isnan().all() and h[T:].isnan().all()

    # fp16 pair: hi = fp16(x), lo = fp16(x - fp16(x)) exactly, with and without the fp32 copy
    x2, hi, lo = _nan(T, H), _nan(T, H, dtype=torch.float16), _nan(T, H, dtype=torch.float16)
    assert lib.sr_test_embed_ln_modernbert(_p(ids), T, H, vocab, _p(table), _p(w), eps, _p(x2), _p(hi), _p(lo)) == 0
    torch.cuda.synchronize()
    assert torch.equal(x2, x[:T])
    assert torch.equal(hi.view(torch.int16), x2.half().view(torch.int16))
    assert torch.equal(lo.view(torch.int16), (x2 - x2.half().float()).half().view(torch.int16))
    hi2, lo2 = _nan(T, H, dtype=torch.float16), _nan(T, H, dtype=torch.float16)
    assert lib.sr_test_embed_ln_modernbert(_p(ids), T, H, vocab, _p(table), _p(w), eps, None, _p(hi2), _p(lo2)) == 0
    torch.cuda.synchronize()
    assert torch.equal(hi2.view(torch.int16), hi.view(torch.int16))
    assert torch.equal(lo2.view(torch.int16), lo.view(torch.int16))
    pair = ro.Ref(ref.value, ref.coef, ref.eps + 2.0 ** -22 * ref.value.abs() + 2.0 ** -25)
    check("embed_ln_modernbert.hl", hi2.double() + lo2.double(), pair)


@pytest.mark.parametrize("H", [384, 768, 1024])
@pytest.mark.parametrize("T", [1, 7, 8, 9, 1037, 65537])
def test_embed_ln_bert(lib, H, T):
    vocab, max_pos, eps = 1000, 512, 1e-12
    g = _gen(T * 11 + H)
    word = _rows(vocab, H, g)
    pos_emb = (0.5 * torch.randn(max_pos, H, device=DEV, generator=g)).contiguous()
    type0 = (0.5 * torch.randn(H, device=DEV, generator=g)).contiguous()
    w = (1.0 + 0.5 * torch.randn(H, device=DEV, generator=g)).contiguous()
    b = (0.5 * torch.randn(H, device=DEV, generator=g)).contiguous()
    ids = _ids(T, vocab, g)
    pos = torch.randint(0, max_pos + 64, (T,), device=DEV, generator=g, dtype=torch.int32)
    edge = torch.tensor([max_pos - 1, max_pos, max_pos + 1, 0, 2 ** 31 - 1], device=DEV, dtype=torch.int32)
    pos[:min(T, 5)] = edge[:min(T, 5)]
    x, h = _nan(T + 8, H), _nan(T + 8, H, dtype=torch.float16)
    assert lib.sr_test_embed_ln_bert(_p(ids), _p(pos), T, H, vocab, max_pos, _p(word), _p(pos_emb), _p(type0), _p(w),
                                     _p(b), eps, _p(x), _p(h)) == 0
    torch.cuda.synchronize()
    ref = ro.embed_ln_bert(ids, pos, word, pos_emb, type0, w, b, eps, max_pos)
    check("embed_ln_bert.x", x[:T], ref)
    check("embed_ln_bert.h", h[:T], ro.f16_out(ref))
    assert x[T:].isnan().all() and h[T:].isnan().all()


# ---- positions and cast ----------------------------------------------------------------------------------------------
def test_positions(lib):
    lens = [1, 0, 5, 128, 129, 0, 3000, 2, 511, 1]
    cu = np.zeros(len(lens) + 1, np.int32)
    cu[1:] = np.cumsum(lens)
    d_cu = torch.from_numpy(cu).to(DEV)
    pos = torch.full((int(cu[-1]) + 4,), -7, device=DEV, dtype=torch.int32)
    assert lib.sr_test_positions(_p(d_cu), len(lens), _p(pos)) == 0
    torch.cuda.synchronize()
    got = pos.cpu().numpy()
    np.testing.assert_array_equal(got[:cu[-1]], ro.positions(cu))
    assert (got[cu[-1]:] == -7).all()


@pytest.mark.parametrize("n", [1, 2, 3, 4, 5, 6, 7, 8, 13, 1001, 768 * 4096 + 1, 768 * 4096 + 2, 768 * 4096 + 3])
def test_cast_f16(lib, n):
    """exact against torch's round-to-nearest, for every n (the tail past the last float4 included)"""
    g = _gen(n)
    special = torch.tensor([65504.0, 65519.0, 65520.0, 7e4, -1e6, 6e-8, 3e-8, 2.9e-8, -1e-6, 6.1e-5, 0.0, -0.0,
                            float("inf"), float("-inf"), 1.0 + 2.0 ** -11, 1.0 + 3 * 2.0 ** -11], device=DEV)
    x = torch.randn(n, device=DEV, generator=g) * torch.exp2(torch.randint(-26, 18, (n,), device=DEV, generator=g).float())
    k = min(n, len(special))
    x[-k:] = special[:k]
    y = torch.full((n + 8,), 0x7E5A, device=DEV, dtype=torch.int16)
    assert lib.sr_test_cast_f16(_p(x), n, _p(y)) == 0
    torch.cuda.synchronize()
    assert torch.equal(y[:n], x.half().view(torch.int16))
    assert (y[n:] == 0x7E5A).all()


# ---- LayerNorm rows --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("H", [384, 768, 1024])
@pytest.mark.parametrize("bias", [False, True])
@pytest.mark.parametrize("y32", ["none", "separate", "alias"])
def test_layernorm(lib, H, bias, y32):
    T, eps = 1037, 1e-5
    g = _gen(H + 2 * bias)
    x = _rows(T, H, g) * 3
    w = torch.randn(H, device=DEV, generator=g)
    b = torch.randn(H, device=DEV, generator=g) if bias else None
    ref = ro.layer_norm(x, w, b, eps, ro.warp_ln_depth(H))
    x0 = x.clone()
    out32 = {"none": None, "separate": _nan(T, H), "alias": x}[y32]
    y16 = _nan(T, H, dtype=torch.float16)
    assert lib.sr_test_layernorm(_p(x), T, H, _p(w), _p(b), eps, _p(out32), _p(y16)) == 0
    torch.cuda.synchronize()
    check("layernorm_rows.h", y16, ro.f16_out(ref))
    if out32 is not None:
        check("layernorm_rows.x", out32, ref)
    if y32 != "alias":
        assert torch.equal(x, x0)


# ---- pooling -----------------------------------------------------------------------------------------------------------
POOL_LENS = [1, 2, 56, 57, 63, 64, 65, 449, 512, 4096, 32768]


def _pool(lib, x, cu, H, mode, w=None, b=None, eps=0.0, div=None, arrived=None):
    B = len(cu) - 1
    d_cu = torch.from_numpy(np.asarray(cu, np.int32)).to(DEV)
    pooled = _nan(B + 1, H)
    part = _nan(B, 8, H)
    arrived = torch.zeros(B, device=DEV, dtype=torch.int32) if arrived is None else arrived
    d_div = None if div is None else torch.from_numpy(np.asarray(div, np.int32)).to(DEV)
    assert lib.sr_test_pool_rows(_p(x), _p(d_cu), B, H, mode, _p(w), _p(b), eps, _p(pooled), _p(part), _p(arrived),
                                 _p(d_div)) == 0
    torch.cuda.synchronize()
    assert (arrived == 0).all(), "arrived must be zero again after the call"
    assert pooled[B].isnan().all()
    return pooled[:B]


def _cu(lens):
    cu = np.zeros(len(lens) + 1, np.int64)
    cu[1:] = np.cumsum(lens)
    return cu


@pytest.mark.parametrize("case", ["mean_ln", "mean", "cls_ln", "cls", "mean_div"])
def test_pool_rows(lib, case):
    H = {"mean_ln": 768, "mean": 1024, "cls_ln": 384, "cls": 768, "mean_div": 384}[case]
    g = _gen(len(case))
    rng = np.random.default_rng(len(case))
    lens = []
    for L in POOL_LENS:   # each long sequence next to short ones
        lens += [L] + list(rng.integers(1, 9, 2))
    cu = _cu(lens)
    x = _rows(int(cu[-1]), H, g)
    mode = 1 if case.startswith("cls") else 0
    w = (1.0 + 0.5 * torch.randn(H, device=DEV, generator=g)) if case.endswith("_ln") else None
    b = (0.5 * torch.randn(H, device=DEV, generator=g)) if case == "cls_ln" else None
    eps = 1e-5 if w is not None else 0.0
    div = [max(1, int(rng.integers(1, L + 1))) for L in lens] if case == "mean_div" else None
    got = _pool(lib, x, cu, H, mode, w, b, eps, div)
    ref = ro.pool_rows(x, cu, mode, w, b, eps, div)
    check(f"pool_rows.{case}", got, ref)
    # a sequence pooled alone equals the same sequence pooled inside the batch, bit for bit
    for i in (POOL_LENS.index(57) * 3, POOL_LENS.index(32768) * 3):
        a, e = int(cu[i]), int(cu[i + 1])
        alone = _pool(lib, x[a:e].contiguous(), [0, e - a], H, mode, w, b, eps, None if div is None else [div[i]])
        assert torch.equal(alone[0], got[i])


def test_pool_rows_back_to_back(lib):
    """two calls on one `arrived` buffer give the same result (the last CTA resets it)"""
    H, lens = 768, [57, 3, 4096, 1, 64, 65]
    cu = _cu(lens)
    x = _rows(int(cu[-1]), H, _gen(5))
    arrived = torch.zeros(len(lens), device=DEV, dtype=torch.int32)
    first = _pool(lib, x, cu, H, 0, arrived=arrived)
    second = _pool(lib, x, cu, H, 0, arrived=arrived)
    assert torch.equal(first, second)
    check("pool_rows.mean", second, ro.pool_rows(x, cu, 0))


# ---- L2 normalisation ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dim", [1, 31, 64, 100, 768])
@pytest.mark.parametrize("norm_eps", [0.0, 1e-12])
def test_l2_normalize(lib, dim, norm_eps):
    H, B = 768, 37
    g = _gen(dim)
    # row scales 1e-12 ... 1e2: at the small end norm_eps moves the result, and an eps inside the sqrt would swamp it
    scale = torch.pow(10.0, torch.linspace(-12, 2, B, device=DEV))
    pooled = (torch.randn(B, H, device=DEV, generator=g) * scale[:, None] / max(dim, 1) ** 0.5).contiguous()
    emb = _nan(B + 1, dim)
    assert lib.sr_test_l2_normalize(_p(pooled), B, H, dim, norm_eps, _p(emb)) == 0
    torch.cuda.synchronize()
    check("l2_normalize_rows", emb[:B], ro.l2_normalize(pooled, dim, norm_eps))
    assert emb[B].isnan().all()


# ---- sequence head ---------------------------------------------------------------------------------------------------
SEQ_MODES = {   # name: (dense_mode, gelu_erf, head_eps)
    "none": (0, 0, 1e-12), "mb_tanh": (1, 0, 1e-12), "mb_erf": (1, 1, 1e-5), "pooler_pt": (2, 0, 1e-12),
    "pooler_p": (3, 0, 1e-12)}


def _head_inputs(B, H, g):
    """half the rows with |x| in [1, 3] (tanh and erf GELU differ most), half 2 +- 0.005 (GELU outputs of variance
    ~5e-5: the head LayerNorm eps shows)"""
    x = (1.0 + 2.0 * torch.rand(B, H, device=DEV, generator=g)) * torch.sign(torch.randn(B, H, device=DEV, generator=g))
    x[1::2] = 2.0 + 0.005 * torch.randn(x[1::2].shape, device=DEV, generator=g)
    return x.contiguous()


def _seq_weights(mode, H, Cn, g):
    dense_mode, _, _ = SEQ_MODES[mode]
    d = {}
    if dense_mode == 1:   # near identity (pre-activations stay where _head_inputs put them), not symmetric
        d["dense_w"] = torch.eye(H, device=DEV) + 0.002 * torch.randn(H, H, device=DEV, generator=g) / H ** 0.5
        d["norm_w"] = 0.5 + torch.rand(H, device=DEV, generator=g)
    elif dense_mode in (2, 3):
        d["dense_w"] = torch.randn(H, H, device=DEV, generator=g) / H ** 0.5 * 0.5
        d["dense_b"] = 0.5 * torch.randn(H, device=DEV, generator=g)
    d["cls_w"] = torch.randn(Cn, H, device=DEV, generator=g) * (2.0 / H ** 0.5)
    d["cls_b"] = torch.randn(Cn, device=DEV, generator=g)
    return {k: v.contiguous() for k, v in d.items()}


def _seq_head(lib, SeqW, pooled, H, mode, wts, argmax_last, Cn):
    dense_mode, gelu_erf, head_eps = SEQ_MODES[mode]
    B = pooled.shape[0]
    sw = SeqW(dense_w=_p(wts.get("dense_w")), dense_b=_p(wts.get("dense_b")), norm_w=_p(wts.get("norm_w")),
              dense_mode=dense_mode, cls_w=_p(wts["cls_w"]), cls_b=_p(wts["cls_b"]), num_classes=Cn,
              argmax_last=argmax_last, gelu_erf=gelu_erf, head_eps=head_eps)
    logits, probs = _nan(B + 1, Cn), _nan(B + 1, Cn)
    cls = torch.full((B + 1,), -7, device=DEV, dtype=torch.int32)
    conf = _nan(B + 1)
    assert lib.sr_test_seq_head(_p(pooled), B, H, C.byref(sw), _p(logits), _p(probs), _p(cls), _p(conf)) == 0
    torch.cuda.synchronize()
    assert logits[B].isnan().all() and probs[B].isnan().all() and int(cls[B]) == -7 and conf[B].isnan()
    return logits[:B], probs[:B], cls[:B], conf[:B]


def _ref_seq(pooled, mode, wts):
    dense_mode, gelu_erf, head_eps = SEQ_MODES[mode]
    return ro.seq_head(pooled, wts["cls_w"], wts["cls_b"], dense_mode=dense_mode, dense_w=wts.get("dense_w"),
                       dense_b=wts.get("dense_b"), norm_w=wts.get("norm_w"), gelu_erf=bool(gelu_erf), head_eps=head_eps)


def _top2_gap_clear(ref):
    """rows whose float64 top-2 gap exceeds the two bounds: the class cannot depend on rounding"""
    v, b = ref.value.cpu(), ref.eps.cpu()
    if v.shape[1] < 2:
        return np.ones(v.shape[0], bool)
    top = v.topk(2, dim=1)
    bt = b.gather(1, top.indices)
    return ((top.values[:, 0] - top.values[:, 1]) > bt.sum(1)).numpy()


@pytest.mark.parametrize("mode", list(SEQ_MODES))
@pytest.mark.parametrize("H", [384, 768, 1024])
@pytest.mark.parametrize("Cn", [1, 2, 3, 14, 33, 100])
def test_seq_head(lib, SeqW, mode, H, Cn):
    g = _gen(H + Cn)
    wts = _seq_weights(mode, H, Cn, g)
    for B in (1, 5, 300):
        argmax_last = (B + Cn) % 2
        pooled = _head_inputs(B, H, g) if mode.startswith("mb") else torch.randn(B, H, device=DEV, generator=g)
        logits, probs, cls, conf = _seq_head(lib, SeqW, pooled, H, mode, wts, argmax_last, Cn)
        rl, rp = _ref_seq(pooled, mode, wts)
        check(f"seq_head.logits.{mode}", logits, rl)
        check(f"seq_head.probs.{mode}", probs, rp)
        pn, cn = probs.cpu().numpy(), cls.cpu().numpy()
        want = np.array([ro.seq_class(r, argmax_last) for r in pn])
        np.testing.assert_array_equal(cn, want)
        assert torch.equal(conf, probs.gather(1, cls.long()[:, None])[:, 0])
        clear = _top2_gap_clear(rp)
        want64 = np.array([ro.seq_class(r, argmax_last) for r in rp.value.cpu().numpy()])
        np.testing.assert_array_equal(cn[clear], want64[clear])


@pytest.mark.parametrize("argmax_last", [0, 1])
@pytest.mark.parametrize("pair", [(0, 1), (3, 13), (5, 13)])
@pytest.mark.parametrize("larger", [None, 8])
def test_seq_head_ties(lib, SeqW, argmax_last, pair, larger):
    H, Cn, B = 768, 14, 4   # (5, 13) = (5, C - 1)
    g = _gen(sum(pair))
    wts = _seq_weights("none", H, Cn, g)
    i, j = pair
    wts["cls_w"][j] = wts["cls_w"][i]
    wts["cls_b"][j] = wts["cls_b"][i] = 6.0
    if larger is not None:
        wts["cls_b"][larger] = 9.0
    pooled = torch.randn(B, H, device=DEV, generator=g) * 0.1
    logits, probs, cls, conf = _seq_head(lib, SeqW, pooled, H, "none", wts, argmax_last, Cn)
    assert torch.equal(logits[:, i], logits[:, j]) and torch.equal(probs[:, i], probs[:, j])
    want = larger if larger is not None else (j if argmax_last else i)
    assert cls.tolist() == [want] * B
    assert torch.equal(conf, probs[:, want])


# ---- token head ------------------------------------------------------------------------------------------------------
TOKEN_PATHS = {   # name: (fp16 dense input, gelu_erf, head_eps, pre-LN)
    "dense_tanh": (True, 0, 1e-12, False), "dense_erf": (True, 1, 1e-5, False), "f32": (False, 0, 0.0, False),
    "f32_ln": (False, 0, 0.0, True)}


def _token_head(lib, path, H, T, Cn, argmax_last, ins, wts, pre_eps=1e-5):
    dense, gelu_erf, head_eps, pre_ln = TOKEN_PATHS[path]
    logits, probs = _nan(T + 1, Cn), _nan(T + 1, Cn)
    pred = torch.full((T + 1,), -7, device=DEV, dtype=torch.int32)
    conf = _nan(T + 1)
    rc = lib.sr_test_token_head(None if dense else _p(ins), _p(ins) if dense else None, T, H, _p(wts.get("norm_w")),
                                _p(wts.get("pre_ln_w")) if pre_ln else None, pre_eps, _p(wts["cls_w"]), _p(wts["cls_b"]),
                                Cn, argmax_last, _p(logits), _p(probs), _p(pred), _p(conf), gelu_erf, head_eps)
    torch.cuda.synchronize()
    return rc, logits, probs, pred, conf


def _token_inputs(path, T, H, g):
    if TOKEN_PATHS[path][0]:
        return _head_inputs(T, H, g).half().contiguous()
    return _rows(T, H, g)


def _token_weights(H, Cn, g):
    return {"norm_w": (0.5 + torch.rand(H, device=DEV, generator=g)).contiguous(),
            "pre_ln_w": (1.0 + 0.5 * torch.randn(H, device=DEV, generator=g)).contiguous(),
            "cls_w": (torch.randn(max(Cn, 1), H, device=DEV, generator=g) * (2.0 / H ** 0.5)).contiguous(),
            "cls_b": torch.randn(max(Cn, 1), device=DEV, generator=g).contiguous()}


def _ref_token(path, H, ins, wts, pre_eps=1e-5):
    dense, gelu_erf, head_eps, pre_ln = TOKEN_PATHS[path]
    kw = dict(dense16=ins, norm_w=wts["norm_w"], gelu_erf=bool(gelu_erf), head_eps=head_eps) if dense else \
        dict(hidden32=ins, pre_ln_w=wts["pre_ln_w"] if pre_ln else None, pre_ln_eps=pre_eps)
    return ro.token_head(wts["cls_w"], wts["cls_b"], H, **kw)


@pytest.mark.parametrize("path", list(TOKEN_PATHS))
@pytest.mark.parametrize("Cn", [1, 2, 9, 31, 32, 33, 64, 65, 200, 256])
def test_token_head(lib, path, Cn):
    for n, T in enumerate((1, 8, 9, 4097)):
        H = (384, 768, 1024)[(n + Cn) % 3]
        argmax_last = (n + Cn) % 2
        g = _gen(Cn * 10 + n)
        wts = _token_weights(H, Cn, g)
        ins = _token_inputs(path, T, H, g)
        rc, logits, probs, pred, conf = _token_head(lib, path, H, T, Cn, argmax_last, ins, wts)
        assert rc == 0
        assert logits[T].isnan().all() and probs[T].isnan().all() and int(pred[T]) == -7 and conf[T].isnan()
        logits, probs, pred, conf = logits[:T], probs[:T], pred[:T], conf[:T]
        rl, rp = _ref_token(path, H, ins, wts)
        check(f"token_head.logits.{path}", logits, rl)
        check(f"token_head.probs.{path}", probs, rp)
        ln, pn = logits.cpu().numpy(), pred.cpu().numpy()
        np.testing.assert_array_equal(pn, [ro.token_pred(r, argmax_last) for r in ln])
        assert torch.equal(conf, probs.gather(1, pred.long()[:, None])[:, 0])
        clear = _top2_gap_clear(rl)
        want64 = np.array([ro.token_pred(r, argmax_last) for r in rl.value.cpu().numpy()])
        np.testing.assert_array_equal(pn[clear], want64[clear])


@pytest.mark.parametrize("argmax_last", [0, 1])
@pytest.mark.parametrize("tied", [(5, 6), (3, 35, 67), (2, 255)])
@pytest.mark.parametrize("larger", [None, 100])
@pytest.mark.parametrize("path", ["f32", "dense_erf"])
def test_token_head_ties(lib, argmax_last, tied, larger, path):
    """ties between lanes of one slot (5, 6), in one lane across slots (3, 35, 67), and across both (2, 255)"""
    H, Cn, T = 384, 256, 9
    g = _gen(sum(tied) + argmax_last)
    wts = _token_weights(H, Cn, g)
    for c in tied[1:]:
        wts["cls_w"][c] = wts["cls_w"][tied[0]]
    wts["cls_b"][list(tied)] = 40.0
    if larger is not None:
        wts["cls_b"][larger] = 60.0
    ins = _token_inputs(path, T, H, g)
    rc, logits, probs, pred, conf = _token_head(lib, path, H, T, Cn, argmax_last, ins, wts)
    assert rc == 0
    for c in tied[1:]:
        assert torch.equal(logits[:T, c], logits[:T, tied[0]])
    want = larger if larger is not None else (max(tied) if argmax_last else min(tied))
    assert pred[:T].tolist() == [want] * T
    assert torch.equal(conf[:T], probs[:T, want])


@pytest.mark.parametrize("Cn", [0, 257])
def test_token_head_refuses(lib, Cn):
    H, T = 768, 9
    g = _gen(Cn)
    wts = _token_weights(H, 257, g)
    ins = _token_inputs("f32", T, H, g)
    rc, logits, probs, pred, conf = _token_head(lib, "f32", H, T, Cn, 0, ins, wts)
    assert rc != 0
    assert logits.isnan().all() and probs.isnan().all() and (pred == -7).all() and conf.isnan().all()
