"""The loaders' refusals without a GPU (sr_model_load_grouped, binding.GroupedModel, and sr_model_load for one
directory): directories that cannot be served are refused from their config.json and safetensors header alone, BEFORE any
device is touched -- so a host without a GPU sees these messages, not the missing device.  And the text ABI's choice
between one grouped model and three slots for merged checkpoints, on the mock engine."""
import ctypes as C
import json
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def _dir(path, cfg, arch="modernbert"):
    """config.json + a safetensors header with the names the loader inspects (tiny tensors: nothing is uploaded)"""
    from safetensors.numpy import save_file
    os.makedirs(path)
    emb = "model.embeddings.tok_embeddings.weight" if arch == "modernbert" else "bert.embeddings.word_embeddings.weight"
    save_file({emb: np.zeros((4, 8), np.float32), "classifier.weight": np.zeros((2, 8), np.float32)},
              os.path.join(path, "model.safetensors"))
    json.dump(cfg.to_json({0: "a", 1: "b"}), open(os.path.join(path, "config.json"), "w"))
    return str(path)


@pytest.fixture()
def dirs(tmp_path):
    from oracle import encoder_oracle as eo
    base = dict(vocab_size=1000, num_hidden_layers=2, max_position_embeddings=1024, pad_token_id=0)
    return {"a": _dir(tmp_path / "a", eo.ModernBertConfig(**base)),
            "b": _dir(tmp_path / "b", eo.ModernBertConfig(**base)),
            "layers": _dir(tmp_path / "layers", eo.ModernBertConfig(**dict(base, num_hidden_layers=3))),
            "theta": _dir(tmp_path / "theta", eo.ModernBertConfig(**dict(base, local_rope_theta=160000.0))),
            "bert": _dir(tmp_path / "bert", eo.BertConfig(vocab_size=1000, num_hidden_layers=2), "bert"),
            "minilm": _dir(tmp_path / "minilm", eo.BertConfig(vocab_size=1000, num_hidden_layers=2, hidden_size=384,
                                                              intermediate_size=1536), "bert"),
            "missing": str(tmp_path / "missing")}


@pytest.mark.parametrize("other,field", [("layers", "num_hidden_layers"), ("theta", "local_rope_theta"), ("bert", "architecture")])
def test_a_config_field_that_differs_is_named(dirs, other, field):
    import semantic_router_b200 as pkg
    with pytest.raises(pkg.SrError, match=f"do not share one encoder shape: {field} is .* in {dirs[other]} and .* in {dirs['a']}"):
        pkg.GroupedModel([dirs["a"], dirs[other]], [0, 0], device=0)


def test_padded_heads_are_refused(dirs):
    import semantic_router_b200 as pkg
    with pytest.raises(pkg.SrError, match="padded-head"):
        pkg.GroupedModel([dirs["minilm"], dirs["minilm"]], [0, 0], device=0)


@pytest.mark.parametrize("n", [0, 9])
def test_task_count_outside_one_to_eight(dirs, n):
    import semantic_router_b200 as pkg
    with pytest.raises(pkg.SrError, match="n_tasks must be 1 to 8"):
        pkg.GroupedModel([dirs["a"]] * n, [0] * n, device=0)


def test_several_bert_tasks_need_whole_128_column_wi_tiles(tmp_path):
    """BERT's Wi has N = intermediate_size, and a grouped GEMM picks a task's matrix only over whole 128-column tiles:
    I = 1088 is refused for two tasks, from config.json alone.  One task reaches the device like any single load."""
    import torch
    import semantic_router_b200 as pkg
    from oracle import encoder_oracle as eo
    cfg = eo.BertConfig(vocab_size=1000, num_hidden_layers=2, intermediate_size=1088)
    d0, d1 = _dir(tmp_path / "bert0", cfg, "bert"), _dir(tmp_path / "bert1", cfg, "bert")
    with pytest.raises(pkg.SrError, match=f"{d0}: intermediate_size 1088 must be a multiple of 128"):
        pkg.GroupedModel([d0, d1], [0, 0], device=0)
    if torch.cuda.is_available():
        return
    with pytest.raises(pkg.SrError, match="no CUDA device"):
        pkg.GroupedModel([d0], [0], device=0)


def test_token_level_count_must_match(dirs):
    import semantic_router_b200 as pkg
    with pytest.raises(pkg.SrError, match="3 token_level values for 2 task checkpoints"):
        pkg.GroupedModel([dirs["a"], dirs["b"]], [0, 1, 0], device=0)


def test_missing_directory(dirs):
    import semantic_router_b200 as pkg
    with pytest.raises(pkg.SrError, match="cannot read " + dirs["missing"] + "/config.json"):
        pkg.GroupedModel([dirs["a"], dirs["missing"]], [0, 0], device=0)


def test_servable_directories_reach_the_device(dirs):
    """the same encoder shape passes every refusal: only then is a device needed (without one it fails like every load)"""
    import torch
    import semantic_router_b200 as pkg
    if torch.cuda.is_available():
        pytest.skip("a device is present")
    with pytest.raises(pkg.SrError, match="no CUDA device"):
        pkg.GroupedModel([dirs["a"], dirs["b"]], [0, 0], device=0)


# ---- sr_model_load: one directory, refused on the host in the same way; its error names the directory once ----------
def _single_load_error(d):
    import semantic_router_b200 as pkg
    h = C.c_void_p()
    assert pkg.lib().sr_model_load(d.encode(), 0, C.byref(h)) != 0
    assert not h.value                                           # no model returned
    return pkg.lib().sr_last_error().decode()


@pytest.mark.parametrize("fields,message", [
    (dict(hidden_size=512, num_attention_heads=8), "hidden_size unsupported"),
    (dict(intermediate_size=1136), "intermediate_size must be a multiple of 64"),
    (dict(hidden_size=384, num_attention_heads=12, intermediate_size=1152), "head_dim 32 unsupported"),
])
def test_single_load_refuses_an_unservable_config(tmp_path, fields, message):
    from oracle import encoder_oracle as eo
    d = _dir(tmp_path / "m", eo.ModernBertConfig(vocab_size=1000, num_hidden_layers=2, max_position_embeddings=1024, pad_token_id=0,
                                                 **fields))
    err = _single_load_error(d)
    assert message in err and err.count(d) == 1


def test_single_load_of_a_missing_directory(dirs):
    err = _single_load_error(dirs["missing"])
    assert "cannot read " + dirs["missing"] + "/config.json" in err and err.count(dirs["missing"]) == 1


@pytest.mark.parametrize("which", ["a", "bert", "minilm"])
def test_single_load_of_a_servable_directory_reaches_the_device(dirs, which):
    """padded-head (MiniLM) encoders included: only the grouped loader refuses them"""
    import torch
    if torch.cuda.is_available():
        pytest.skip("a device is present")
    assert "no CUDA device" in _single_load_error(dirs[which])


# ---- text ABI on the mock engine: merged checkpoints as one grouped model, or three slots ----------------------------
@pytest.fixture(scope="module")
def mock_lib(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    w = tmp_path_factory.mktemp("grouped_mock")
    path = str(w / "libcandle_mock.so")
    r = subprocess.run(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-o", path, "-x", "c++", "semantic-router_b200/csrc/abi.cu",
                        "-x", "none", "semantic-router_b200/csrc/tokenizer.cc", "tools/abi_sanitize/mock_engine.cc", "-lpthread"],
                       cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    return path, w


_MOCK_RUN = r"""
import ctypes as C, json, os, sys
sys.path.insert(0, os.path.join({root!r}, "tests"))
from test_multi_device_dispatch_mock import LBatch, _arr
lib, dirs, texts = sys.argv[1], json.loads(sys.argv[2]), json.loads(sys.argv[3])
L = C.CDLL(lib)
L.init_lora_unified_classifier.argtypes = [C.c_char_p] * 4 + [C.c_bool]; L.init_lora_unified_classifier.restype = C.c_bool
L.classify_batch_with_lora.argtypes = [C.POINTER(C.c_char_p), C.c_int]; L.classify_batch_with_lora.restype = LBatch
L.sr_mock_device_calls.argtypes = [C.c_int]; L.sr_mock_device_calls.restype = C.c_longlong
assert L.init_lora_unified_classifier(*[d.encode() for d in dirs], b"modernbert", False)
r = L.classify_batch_with_lora(_arr(texts), len(texts))
rows = []
for i in range(r.batch_size):
    p = r.pii_results[i]
    rows.append([r.intent_results[i].category.decode(), r.intent_results[i].confidence.hex(), p.has_pii,
                 [p.pii_types[k].decode() for k in range(p.num_pii_types)], p.confidence.hex(),
                 r.security_results[i].is_jailbreak, r.security_results[i].threat_type.decode(), r.security_results[i].confidence.hex()])
print("RESULT " + json.dumps({{"rows": rows, "calls": L.sr_mock_device_calls(0)}}))
"""


def _mock_run(lib, dirs, texts, **env_set):
    env = {k: v for k, v in os.environ.items()
           if k not in ("SR_MOCK_DEVICES", "SR_B200_DEVICES", "SR_B200_DEVICE", "SR_MOCK_LORA_SHARED", "SR_B200_LORA_SHARED", "SR_MOCK_GROUPED")}
    env.update(env_set)
    r = subprocess.run([sys.executable, "-c", _MOCK_RUN.format(root=ROOT), lib, json.dumps(dirs), json.dumps(texts)],
                       env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-3000:]
    return json.loads([x for x in r.stdout.splitlines() if x.startswith("RESULT ")][-1][len("RESULT "):])


def test_text_abi_groups_merged_checkpoints_like_three_slots(mock_lib):
    """Merged checkpoints (no adapters): the ABI takes the grouped loader -- pieces of at most 256 / 3 texts, three heads
    per piece -- and answers exactly like three slots; SR_B200_LORA_SHARED=0, a grouped loader that refuses, or
    tokenizers that differ between the directories keep the three slots."""
    from oracle import synth, tokenizer_fixtures as tf
    lib, w = mock_lib
    pii = synth.pii_id2label()

    def mk(name, labels, tok="modernbert"):
        d = w / name
        d.mkdir()
        tf.BUILDERS[tok](str(d / "tokenizer.json"))
        json.dump({"model_type": "modernbert", "max_position_embeddings": 1024,
                   "id2label": {str(i): l for i, l in enumerate(labels)}}, open(d / "config.json", "w"))
        return str(d)
    dirs = [mk("intent", [f"cat{i}" for i in range(14)]), mk("pii", [pii[i] for i in range(len(pii))]), mk("sec", ["safe", "jailbreak"])]
    texts = [f"text {i} " + "john@example.com " * (i % 4) + "filler " * (i % 11) for i in range(200)]
    grouped = _mock_run(lib, dirs, texts, SR_MOCK_GROUPED="1")
    slots = _mock_run(lib, dirs, texts, SR_MOCK_GROUPED="1", SR_B200_LORA_SHARED="0")
    refused = _mock_run(lib, dirs, texts)
    assert grouped["rows"] == slots["rows"] == refused["rows"]
    assert slots["calls"] == refused["calls"]
    # grouped: >= ceil(200 / 85) pieces, one engine call per head of each (the mock answers head by head)
    assert grouped["calls"] >= 9 and grouped["calls"] % 3 == 0 and grouped["calls"] != slots["calls"]
    other_tok = [dirs[0], dirs[1], mk("sec_bert_tok", ["safe", "jailbreak"], "bert")]
    assert _mock_run(lib, other_tok, texts, SR_MOCK_GROUPED="1")["calls"] == slots["calls"]
