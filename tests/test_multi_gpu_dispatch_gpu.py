"""In-library multi-GPU dispatch on real hardware (needs >= 2 visible GPUs; skipped on one).
The reference router is ONE process (a goroutine per signal per request, classifier_signal_dispatch.go:114-129); the
library replicates each slot on every visible GPU and spreads callers / batch pieces over them (abi_core.h).  The C
harness plays the cgo side with 64 OS threads: every answer equals the single-threaded one to 1e-6 whichever GPU served
it, and every GPU took a share of the requests."""
import json
import os
import subprocess
import tempfile

import pytest

from oracle import encoder_oracle as eo, synth, tokenizer_fixtures as tf

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_64_threads_keep_every_gpu_busy(srlib, cuda):
    import torch
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("one GPU visible")
    exe = os.path.join(tempfile.mkdtemp(prefix="srb_harness_"), "abi_stress")
    subprocess.check_call(["gcc", "-O2", "-o", exe, os.path.join(ROOT, "tests", "c_harness", "abi_stress.c"), "-ldl", "-lpthread", "-lm"])
    cfg = eo.ModernBertConfig(vocab_size=700, num_hidden_layers=4, max_position_embeddings=1024, pad_token_id=3)
    w = synth.make_modernbert_weights(cfg, 14, seed=41)
    d = tempfile.mkdtemp(prefix="srb_abi_mgpu_")
    tf.build_modernbert(os.path.join(d, "tokenizer.json"))
    synth.write_model_dir(d, cfg, w, {i: f"cat{i}" for i in range(14)})
    env = {k: v for k, v in os.environ.items() if k not in ("SR_B200_DEVICE", "SR_B200_DEVICES")}
    r = subprocess.run([exe, srlib.LIB_PATH, d, "64", "40"], capture_output=True, text=True, timeout=600, env=env)
    assert r.returncode == 0, r.stdout + r.stderr
    out = json.loads(r.stdout.strip().splitlines()[-1])
    print(out)
    assert out["errors"] == 0 and out["requests"] == 64 * 40
    per = out["device_requests"][:n]
    assert sum(per) >= 64 * 40 and min(per) >= 64 * 40 // (4 * n), per     # every GPU served a real share
    assert all(x == 0 for x in out["device_requests"][n:])
    # pinned to one device: the others stay idle
    r = subprocess.run([exe, srlib.LIB_PATH, d, "8", "10"], capture_output=True, text=True, timeout=600,
                       env=dict(env, SR_B200_DEVICES="1"))
    assert r.returncode == 0, r.stdout + r.stderr
    out = json.loads(r.stdout.strip().splitlines()[-1])
    assert out["errors"] == 0 and out["device_requests"][0] == 0 and out["device_requests"][1] >= 80
