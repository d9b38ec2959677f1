"""Secondary measurement (SURVEY section 8 f3): three LoRA tasks (intent / PII tokens / security) over ONE ModernBERT-base --
a batch through the shared-base pass (sr_classify_lora_shared_ids: one encoder pass over three copies of the rows, each
256-row block of a projection GEMM multiplied with its task's merged weights) against the three-slot path (three models with the adapters folded at load, three passes),
through the host-buffer C ABI.  Synthetic weights; prints one JSON line."""
import json, os, sys, tempfile, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import semantic_router_b200 as pkg
from oracle import encoder_oracle as eo, synth

RANK, ALPHA = 16, 32.0
TASKS = [(14, 0), (35, 1), (2, 0)]    # classes, token-level
cfg = eo.ModernBertConfig(vocab_size=50368, num_hidden_layers=22, max_position_embeddings=1024, pad_token_id=0)
root = os.path.join(tempfile.gettempdir(), "srb_bench_lora_shared")
dirs = [os.path.join(root, f"task{t}") for t in range(3)]
if not os.path.exists(os.path.join(root, ".complete")):
    base = synth.make_modernbert_weights(cfg, 14, seed=1234)
    H, I = cfg.hidden_size, cfg.intermediate_size
    for t, (ncls, _tok) in enumerate(TASKS):
        w = dict(base)
        head = synth.make_modernbert_weights(eo.ModernBertConfig(vocab_size=8, num_hidden_layers=0), ncls, seed=50 + t)
        for k in ("head.dense.weight", "head.norm.weight", "classifier.weight", "classifier.bias"):
            w[k] = head[k]
        rng = np.random.default_rng(60 + t)
        for li in range(cfg.num_hidden_layers):
            for name, (o, i) in (("attn.Wqkv", (3 * H, H)), ("attn.Wo", (H, H)), ("mlp.Wi", (2 * I, H)), ("mlp.Wo", (H, I))):
                stem = f"model.layers.{li}.{name}"
                w[stem + ".lora_A.weight"] = (rng.standard_normal((RANK, i)) * 0.02).astype(np.float32)
                w[stem + ".lora_B.weight"] = (rng.standard_normal((o, RANK)) * 0.02).astype(np.float32)
        synth.write_model_dir(dirs[t], cfg, w, {i: f"c{i}" for i in range(ncls)})
        json.dump({"rank": RANK, "alpha": ALPHA}, open(os.path.join(dirs[t], "lora_config.json"), "w"))
    open(os.path.join(root, ".complete"), "w").write("ok")

shared = pkg.LoraSharedModel(dirs, [t[1] for t in TASKS], device=0)
slots = [pkg.Model(d, device=0) for d in dirs]
rng = np.random.default_rng(7)


def three(seqs):
    return [slots[t].classify_tokens_ids(seqs) if TASKS[t][1] else slots[t].classify_ids(seqs) for t in range(3)]


def timed(fn, n):
    for _ in range(max(3, n // 10)):
        fn()
    ts = []
    for _ in range(n):
        t0 = time.perf_counter(); fn(); ts.append(time.perf_counter() - t0)
    ts = np.sort(np.array(ts)) * 1e3
    return {"p50_ms": round(float(ts[len(ts) // 2]), 3), "p95_ms": round(float(ts[int(len(ts) * 0.95)]), 3)}


out = {"workload": f"ModernBERT-base (22 layers), 3 LoRA tasks rank {RANK} on Wqkv / Wo / Wi / Wo-mlp, host-buffer C ABI",
       "weights_resident": {"shared_pass": "base + three merged copies of the projections, stacked", "three_slots": "three merged models"}}
for B, S, n in ((1, 128, 200), (1, 512, 200), (8, 512, 60), (64, 512, 20)):
    seqs = [rng.integers(5, cfg.vocab_size, size=S, dtype=np.int32) for _ in range(B)]
    a = timed(lambda: shared.classify_shared_ids(seqs), n)
    b = timed(lambda: three(seqs), n)
    ref = three(seqs)
    probs, _, _ = shared.classify_shared_ids(seqs)
    dmax = max(float(np.abs(probs[t] - ref[t]["probs"]).max()) for t in range(3))
    out[f"b{B}_s{S}"] = {"shared_pass": a, "three_slots": b, "speedup_p50": round(b["p50_ms"] / a["p50_ms"], 2),
                         "max_dprob_vs_three_slots": dmax}
print(json.dumps(out))
