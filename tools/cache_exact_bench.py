"""Default cache against exact cache (sr_cache_create_exact) on BASELINE cfg 4: 1 M x 768 unit rows, k 8, b 1024 and b 1.

Both caches hold the same rows; the timed calls alternate between them (sr_cache_topk, host queries in, host results out,
wall clock around each synchronous call).  Prints one JSON line with the median and spread per (cache, b), the exact
cache's fallback queries, the device memory each cache added, and the card's name and power limit read in the same run.

    python tools/cache_exact_bench.py [--n 1048576] [--reps 10] [--rule 0]
"""
import argparse
import importlib
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1 << 20)
    ap.add_argument("--d", type=int, default=768)
    ap.add_argument("--k", type=int, default=8)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--rule", type=int, default=0)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark measures the GPU only")
    pkg = importlib.import_module("semantic-router_b200")
    from oracle import synth
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    rng = np.random.default_rng(4)
    rows = synth.make_cache(rng, a.n, a.d)
    queries = {b: synth.make_queries(rng, rows, b)[0].astype(np.float32) for b in (1024, 1)}

    def used():
        torch.cuda.synchronize()
        free, total = torch.cuda.mem_get_info()
        return total - free

    m0 = used()
    caches = {"default": pkg.Cache(a.n, a.d)}
    caches["default"].add(rows)
    m1 = used()
    caches["exact"] = pkg.Cache(a.n, a.d, exact=True, sum_rule=a.rule)
    caches["exact"].add(rows)
    m2 = used()
    # "scan k'": the default cache at the exact cache's candidate count k', i.e. the exact cache's fp16 candidate scan alone
    runs = {"default": ("default", a.k), "exact": ("exact", a.k), "scan k'": ("default", None)}
    times = {(name, b): [] for name in runs for b in queries}
    fallback, kc = {}, {}
    for b, q in queries.items():
        caches["exact"].topk(q, a.k)
        _, _, _, kc[b], fallback[b] = caches["exact"].exact_stats(b)
        for name, (which, k) in runs.items():   # warm-up: module load, workspace growth
            caches[which].topk(q, k or kc[b])
        for _ in range(a.reps):
            for name, (which, k) in runs.items():
                t0 = time.perf_counter()
                caches[which].topk(q, k or kc[b])
                times[(name, b)].append((time.perf_counter() - t0) * 1e3)
    out = {
        "card": card, "n": a.n, "d": a.d, "k": a.k, "rule": a.rule,
        "ms": {f"{name} b{b}": {"median": float(np.median(v)), "min": float(np.min(v)), "max": float(np.max(v))}
               for (name, b), v in times.items()},
        "exact_fallback_queries": {f"b{b}": v for b, v in fallback.items()},
        "exact_candidates": {f"b{b}": v for b, v in kc.items()},
        "device_bytes_default_cache": m1 - m0,
        "device_bytes_exact_cache": m2 - m1,
    }
    print(json.dumps(out))
    for c in caches.values():
        c.close()


if __name__ == "__main__":
    main()
