"""Grouped pass against separate slots (sr_b200.h: sr_model_load_grouped): 3 and 5 task checkpoints of ModernBERT-base
(22 layers) -- heads of 14 (sequence), 35 (token), 2, 2 and 4 (sequence) classes -- in two forms: merged from one base
(only the four projections differ, as merged LoRA models do) and fully distinct (every tensor differs).  A batch of B
prompts of S tokens goes once through the grouped model (one encoder pass over n_tasks copies of the rows) and once
through n_tasks separately loaded models, through the host-buffer C ABI.  Reports p50 / p95 per call and the device bytes
each arrangement holds.  Synthetic weights; prints one JSON line."""
import json, os, sys, tempfile, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import semantic_router_b200 as pkg
from oracle import encoder_oracle as eo, synth

TASKS = [(14, 0), (35, 1), (2, 0), (2, 0), (4, 0)]    # classes, token-level
SHAPES = ((1, 128, 200), (1, 512, 200), (8, 512, 60), (64, 512, 20))   # B, S, timed calls
cfg = eo.ModernBertConfig(vocab_size=50368, num_hidden_layers=22, max_position_embeddings=1024, pad_token_id=0)
root = os.path.join(tempfile.gettempdir(), "srb_bench_grouped")
H, I = cfg.hidden_size, cfg.intermediate_size


def write_sets():
    """merged{t}: one base, per-task projections (base + a rank-16 update) and heads; distinct{t}: every tensor its own"""
    if os.path.exists(os.path.join(root, ".complete")):
        return
    base = synth.make_modernbert_weights(cfg, 0, seed=1234, with_head=False)
    for t, (ncls, _tok) in enumerate(TASKS):
        head = synth.make_modernbert_weights(eo.ModernBertConfig(vocab_size=8, num_hidden_layers=0), ncls, seed=50 + t)
        heads = {k: head[k] for k in ("head.dense.weight", "head.norm.weight", "classifier.weight", "classifier.bias")}
        w = dict(base)
        w.update(heads)
        rng = np.random.default_rng(60 + t)
        for li in range(cfg.num_hidden_layers):
            for name, (o, i) in (("attn.Wqkv", (3 * H, H)), ("attn.Wo", (H, H)), ("mlp.Wi", (2 * I, H)), ("mlp.Wo", (H, I))):
                stem = f"model.layers.{li}.{name}.weight"
                A = rng.standard_normal((16, i), dtype=np.float32) * np.float32(0.02)
                B = rng.standard_normal((o, 16), dtype=np.float32) * np.float32(0.02)
                w[stem] = w[stem] + np.float32(2.0) * (B @ A)
        labels = {i: f"c{i}" for i in range(ncls)}
        half = lambda ws: {k: v.astype(np.float16) for k, v in ws.items()}   # fp16 checkpoints: half the disk
        synth.write_model_dir(os.path.join(root, f"merged{t}"), cfg, half(w), labels)
        d = synth.make_modernbert_weights(cfg, 0, seed=700 + t, with_head=False)
        d.update(heads)
        synth.write_model_dir(os.path.join(root, f"distinct{t}"), cfg, half(d), labels)
    open(os.path.join(root, ".complete"), "w").write("ok")


def timed(fn, n):
    for _ in range(max(3, n // 10)):
        fn()
    ts = []
    for _ in range(n):
        t0 = time.perf_counter(); fn(); ts.append(time.perf_counter() - t0)
    ts = np.sort(np.array(ts)) * 1e3
    return {"p50_ms": round(float(ts[len(ts) // 2]), 3), "p95_ms": round(float(ts[int(len(ts) * 0.95)]), 3)}


def main():
    write_sets()
    out = {"workload": "ModernBERT-base (22 layers), host-buffer C ABI; grouped pass vs one slot per task",
           "tasks": [{"classes": c, "token_level": bool(tok)} for c, tok in TASKS]}
    try:
        import subprocess
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        out["gpu"] = q.stdout.strip()
    except Exception as e:   # the numbers still stand; the GPU line is then missing
        out["gpu"] = f"unavailable: {e}"
    rng = np.random.default_rng(7)
    for n in (3, 5):
        tasks = TASKS[:n]
        for form in ("merged", "distinct"):
            dirs = [os.path.join(root, f"{form}{t}") for t in range(n)]
            grouped = pkg.GroupedModel(dirs, [t[1] for t in tasks], device=0)
            slots = [pkg.Model(d, device=0) for d in dirs]

            def separate(seqs):
                return [slots[t].classify_tokens_ids(seqs) if tasks[t][1] else slots[t].classify_ids(seqs) for t in range(n)]
            key = f"{n}_tasks_{form}"
            res = {"device_bytes": {"grouped": grouped.device_bytes(), "separate_slots": sum(s.device_bytes() for s in slots)}}
            for B, S, iters in SHAPES:
                seqs = [rng.integers(5, cfg.vocab_size, size=S, dtype=np.int32) for _ in range(B)]
                a = timed(lambda: grouped.classify_shared_ids(seqs), iters)
                b = timed(lambda: separate(seqs), iters)
                ref = separate(seqs)
                probs, _, _ = grouped.classify_shared_ids(seqs)
                same = all(np.array_equal(probs[t], ref[t]["probs"]) for t in range(n))
                res[f"b{B}_s{S}"] = {"grouped": a, "separate_slots": b, "speedup_p50": round(b["p50_ms"] / a["p50_ms"], 2),
                                     "bitwise_equal_to_slots": same}
            out[key] = res
            grouped.close()
            for s in slots:
                s.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
