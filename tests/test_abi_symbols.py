"""The C-ABI library loads without a GPU and exports every symbol include/*.h declares (no compute calls)."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared(path):
    src = open(path).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    src = re.sub(r"//[^\n]*", "", src)
    names = set()
    for m in re.finditer(r"\b([A-Za-z_][A-Za-z0-9_]*)\s*\([^;{}]*\)\s*;", src):
        n = m.group(1)
        if n not in ("__attribute__", "visibility", "defined"):
            names.add(n)
    return names


@pytest.fixture(scope="module")
def lib():
    import semantic_router_b200 as pkg
    return pkg.load_library()


ONNX_HEADER = "onnx_semantic_router.h"   # bound by the twin library (same names, other signatures)
HOOKS_HEADER = "sr_b200_testhooks.h"     # exported by the *_testhooks.so twins only


def test_every_declared_symbol_is_exported(lib):
    import semantic_router_b200 as pkg
    inc = os.path.join(ROOT, "include")
    product = ctypes.CDLL(pkg.LIB_PATH)            # a fresh handle: `lib` carries the hook attributes binding.py attaches
    hooks = ctypes.CDLL(pkg.HOOKS_LIB_PATH)
    missing = []
    total = 0
    for h in sorted(os.listdir(inc)):
        if not h.endswith(".h") or h == ONNX_HEADER:
            continue
        for name in sorted(_declared(os.path.join(inc, h))):
            total += 1
            if not hasattr(hooks if h == HOOKS_HEADER else product, name):
                missing.append(f"{h}:{name}")
            if h != HOOKS_HEADER and not hasattr(hooks, name):
                missing.append(f"testhooks twin lacks {h}:{name}")
    assert total > 30
    assert not missing, missing


def test_product_libraries_export_only_their_c_abi():
    """Dynamic symbol table of the two product libraries == the C functions their headers declare: no sr_test_* hooks,
    no weak std:: template instantiations, no engine internals (the link uses a version script built from include/)."""
    import subprocess
    import semantic_router_b200 as pkg
    inc = os.path.join(ROOT, "include")
    libdir = os.path.dirname(pkg.LIB_PATH)
    for so, headers in (("libcandle_semantic_router.so", ["candle_semantic_router.h", "unified_classifier_abi.h", "sr_b200.h"]),
                        ("libonnx_semantic_router.so", ["onnx_semantic_router.h", "unified_classifier_abi.h", "sr_b200.h"])):
        out = subprocess.run(["nm", "-D", "--defined-only", os.path.join(libdir, so)], capture_output=True, text=True, check=True).stdout
        syms = {l.split()[-1]: l.split()[-2] for l in out.splitlines() if len(l.split()) >= 3}
        declared = set()
        for h in headers:
            declared |= _declared(os.path.join(inc, h))
        assert not [s for s in syms if s.startswith("sr_test_")], so
        assert not [s for s, t in syms.items() if t in ("W", "V", "w", "v")], so     # no weak (C++ library) symbols
        extra = sorted(set(syms) - declared)
        assert not extra, (so, extra[:20])


def test_onnx_twin_exports_its_header():
    """libonnx_semantic_router.so: every symbol of include/onnx_semantic_router.h (onnx-binding/semantic-router.go:98-140)."""
    import semantic_router_b200 as pkg
    twin = ctypes.CDLL(os.path.join(os.path.dirname(pkg.LIB_PATH), "libonnx_semantic_router.so"))
    names = _declared(os.path.join(ROOT, "include", ONNX_HEADER))
    assert len(names) >= 25, sorted(names)
    missing = [n for n in sorted(names) if not hasattr(twin, n)]
    assert not missing, missing
    # and it is a separate ABI: no candle-only entry points leak into it
    assert not hasattr(twin, "init_modernbert_classifier")
    # no model loaded: the documented failure values, not a crash
    twin.is_classifier_loaded.restype = ctypes.c_bool
    assert twin.is_classifier_loaded(b"intent") is False
    twin.is_mmbert_model_initialized.restype = ctypes.c_bool
    assert twin.is_mmbert_model_initialized() is False


def test_both_libraries_cover_the_go_preambles():
    """Every C function the reference's Go files declare in their cgo preambles (tests/golden/go_externs.json, parsed from
    candle-binding/semantic-router.go:27-453, onnx-binding/semantic-router.go:9-141 and
    pkg/classification/unified_classifier.go:5-82 by tools/gen_go_externs.py) resolves in the library Go would link:
    candle + unified in libcandle_semantic_router, onnx + unified in libonnx_semantic_router (-tags=onnx)."""
    import json
    import semantic_router_b200 as pkg
    ext = json.load(open(os.path.join(ROOT, "tests", "golden", "go_externs.json")))
    assert (len(ext["candle"]["externs"]), len(ext["onnx"]["externs"]), len(ext["unified"]["externs"])) == (114, 25, 7)
    libdir = os.path.dirname(pkg.LIB_PATH)
    candle = ctypes.CDLL(os.path.join(libdir, "libcandle_semantic_router.so"))
    onnx = ctypes.CDLL(os.path.join(libdir, "libonnx_semantic_router.so"))
    for lib_, groups in ((candle, ("candle", "unified")), (onnx, ("onnx", "unified"))):
        missing = [f"{g}:{n}" for g in groups for n in ext[g]["externs"] if not hasattr(lib_, n)]
        assert not missing, missing
    # the unified entries of the ONNX twin answer with the Go-declared failure values before any init
    class LB(ctypes.Structure):
        _fields_ = [("i", ctypes.c_void_p), ("p", ctypes.c_void_p), ("s", ctypes.c_void_p), ("batch_size", ctypes.c_int),
                    ("avg_confidence", ctypes.c_float)]
    onnx.classify_batch_with_lora.restype = LB
    onnx.classify_batch_with_lora.argtypes = [ctypes.POINTER(ctypes.c_char_p), ctypes.c_int]
    arr = (ctypes.c_char_p * 1)(b"hello")
    r = onnx.classify_batch_with_lora(arr, 1)
    assert r.batch_size == 0 and not r.i       # unified_classifier.go:309-311: batch_size <= 0 is the failure signal


def test_fails_loudly_without_gpu_or_model(lib):
    import semantic_router_b200 as pkg
    with pytest.raises(pkg.SrError):
        pkg.Model("/nonexistent/dir", device=0)


def test_adapter_probe_and_shared_loader_without_gpu(lib, tmp_path):
    """sr_checkpoint_has_adapters is host code (safetensors header): 1 / 0 / -1; the shared-LoRA loader refuses checkpoints over
    different bases or without adapters BEFORE it touches a device, and without an sm_90 device it fails loudly like every
    other load (no CPU path)."""
    import numpy as np
    import semantic_router_b200 as pkg
    from safetensors.numpy import save_file
    base = {"model.embeddings.tok_embeddings.weight": np.ones((4, 8), np.float32), "model.layers.0.attn.Wo.weight": np.zeros((8, 8), np.float32),
            "classifier.weight": np.zeros((2, 8), np.float32)}
    lora = dict(base)
    lora["model.layers.0.attn.Wo.lora_A.weight"] = np.zeros((2, 8), np.float32)
    lora["model.layers.0.attn.Wo.lora_B.weight"] = np.zeros((8, 2), np.float32)
    other = dict(lora)
    other["model.embeddings.tok_embeddings.weight"] = np.full((4, 8), 2.0, np.float32)
    dirs = {}
    for name, w in (("merged", base), ("lora", lora), ("lora2", lora), ("other", other)):
        d = tmp_path / name
        d.mkdir()
        save_file(w, str(d / "model.safetensors"))
        dirs[name] = str(d)
    L = pkg.lib()
    assert L.sr_checkpoint_has_adapters(dirs["merged"].encode()) == 0
    assert L.sr_checkpoint_has_adapters(dirs["lora"].encode()) == 1
    assert L.sr_checkpoint_has_adapters(str(tmp_path / "missing").encode()) == -1
    with pytest.raises(pkg.SrError, match="share one base"):
        pkg.LoraSharedModel([dirs["lora"], dirs["other"]], [0, 0], device=0)
    with pytest.raises(pkg.SrError, match="no lora_A"):
        pkg.LoraSharedModel([dirs["merged"], dirs["merged"]], [0, 0], device=0)
    import torch
    if not torch.cuda.is_available():
        with pytest.raises(pkg.SrError):                         # same base, adapters present: now it needs the device
            pkg.LoraSharedModel([dirs["lora"], dirs["lora2"]], [0, 0], device=0)


def test_host_merge_topk_matches_oracle():
    import numpy as np
    import semantic_router_b200 as pkg
    from oracle import cache_oracle as co
    rng = np.random.default_rng(0)
    g, b, k = 4, 9, 8
    idx, sc = [], []
    for s in range(g):
        sco = -np.sort(-rng.random((b, k)).astype(np.float32), axis=1)
        sco[:, 5:] = sco[:, 4:5]                       # ties inside a shard
        ii = np.sort(rng.choice(1000, size=(b, k), replace=False), axis=1).astype(np.int32) + 1000 * s
        if s == 2:
            ii[:, 6:] = -1; sco[:, 6:] = -np.inf      # short shard
        idx.append(ii); sc.append(sco)
    mi, ms = pkg.merge_topk(idx, sc)
    oi, os_ = co.merge_topk(idx, sc, k)
    assert (mi == oi).all() and np.array_equal(ms, os_)


def test_safetensors_reader_survives_malformed_files(lib, tmp_path):
    """The safetensors reader of the product library (engine.cu: SafeTensors::open) is reached without a GPU through
    sr_checkpoint_has_adapters: truncated files, header lengths beyond the file, non-JSON headers, offsets outside the data
    section, deeply nested JSON and random bytes must come back as -1 (unreadable) or 0 / 1 -- never crash the process that
    hosts the router (the reference loads the same files through the `safetensors` crate, which validates likewise)."""
    import json
    import struct
    import numpy as np
    import semantic_router_b200 as pkg
    L = pkg.lib()
    rng = np.random.default_rng(5)

    def probe(blob):
        d = tmp_path / f"case{probe.n}"
        probe.n += 1
        d.mkdir()
        (d / "model.safetensors").write_bytes(blob)
        return L.sr_checkpoint_has_adapters(str(d).encode())
    probe.n = 0

    def st(header, data=b"", hlen=None):
        h = json.dumps(header).encode() if not isinstance(header, bytes) else header
        return struct.pack("<Q", len(h) if hlen is None else hlen) + h + data

    good = {"a.lora_A.weight": {"dtype": "F32", "shape": [2, 2], "data_offsets": [0, 16]}}
    assert probe(st(good, b"\0" * 16)) == 1
    assert probe(st({"w": {"dtype": "F32", "shape": [1], "data_offsets": [0, 4]}}, b"\0" * 4)) == 0
    assert probe(b"") == -1 and probe(b"\x01\x02\x03") == -1                                    # shorter than the length word
    assert probe(st(good, b"\0" * 16, hlen=1 << 60)) == -1                                       # header longer than the file
    assert probe(st(good, b"\0" * 16, hlen=(1 << 64) - 1)) == -1
    assert probe(st(b"not json at all {{{", b"")) == -1
    assert probe(st(b"[1, 2, 3]")) == -1                                                         # JSON, but not an object
    assert probe(st({"a.lora_A.weight": {"dtype": "F32", "shape": [2, 2], "data_offsets": [0, 1 << 40]}}, b"\0" * 16)) == -1
    assert probe(st({"a.lora_A.weight": {"dtype": "F32", "shape": [2, 2], "data_offsets": [32, 16]}}, b"\0" * 64)) == -1
    assert probe(st({"a.lora_A.weight": {"dtype": "F32", "shape": [2, 2], "data_offsets": [-8, 8]}}, b"\0" * 64)) == -1
    assert probe(st(b'{"a":' * 5000 + b"1" + b"}" * 5000)) == -1                                 # nesting beyond the parser's depth limit
    assert probe(st({"__metadata__": {"format": "pt"}, "x.lora_A.weight": {"dtype": "F16", "shape": [1, 8], "data_offsets": [0, 16]}}, b"\0" * 16)) == 1
    for _ in range(200):                                                                         # random mutations of a valid file
        blob = bytearray(st(good, b"\0" * 16))
        for _ in range(int(rng.integers(1, 6))):
            blob[int(rng.integers(0, len(blob)))] = int(rng.integers(0, 256))
        if rng.random() < 0.3:
            blob = blob[:int(rng.integers(0, len(blob)))]
        assert probe(bytes(blob)) in (-1, 0, 1)
    for _ in range(50):
        assert probe(rng.integers(0, 256, size=int(rng.integers(0, 400)), dtype=np.uint8).tobytes()) in (-1, 0, 1)
