"""BASELINE cfg 4 sharded over G GPUs (SURVEY section 8e), default cache against exact cache: every rank holds its
shard_range of the 1 M x 768 unit rows twice, in a default cache and in an exact cache (sr_cache_create_exact), and runs
the whole device-resident lookup of sharding.sharded_topk_dev -- scan its shard, pack, one NCCL all-gather of 8-byte
entries, merge -- with fp16 queries on the default cache (sr_cache_topk_packed_dev) and fp32 queries on the exact cache
(sr_cache_topk_packed_f32_dev), alternating the two, at b 1024 and b 1, k 8.  Each lookup is timed on rank 0 by the wall
clock around the call and a device synchronise.  Rank 0 prints one JSON line: the median and spread per (cache, b), each
rank's fallback queries at each b, whether the merged exact ids and score bits equal an unsharded exact cache's
sr_cache_topk for the same queries on rank 0's GPU, and the card's name and power limit read in the same run.

    python -m torch.distributed.run --nnodes=1 --nproc-per-node G --master-addr 127.0.0.1 \\
        tools/cache_exact_sharded_bench.py [--n 1048576] [--reps 10] [--rule 0]
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
    import torch.distributed as dist
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark measures the GPU only")
    pkg = importlib.import_module("semantic-router_b200")
    sh = importlib.import_module("semantic-router_b200.sharding")
    from oracle import synth
    rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    local = int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(local)],
                          capture_output=True, text=True).stdout.strip()
    rng = np.random.default_rng(4)                                   # the same rows and queries on every rank
    rows = synth.make_cache(rng, a.n, a.d)
    queries = {b: synth.make_queries(rng, rows, b)[0].astype(np.float32) for b in (1024, 1)}
    lo, hi = sh.shard_range(a.n, rank, world)
    caches = {"default": pkg.Cache(hi - lo, a.d, device=local, id_offset=lo),
              "exact": pkg.Cache(hi - lo, a.d, device=local, id_offset=lo, exact=True, sum_rule=a.rule)}
    for c in caches.values():
        c.add(rows[lo:hi])
    dq = {b: {"default": torch.from_numpy(q).cuda().half(), "exact": torch.from_numpy(q).cuda()}
          for b, q in queries.items()}
    times = {(name, b): [] for name in caches for b in queries}
    fallback, merged = {}, {}
    for b in queries:
        for name, c in caches.items():                               # warm-up: module load, scratch growth
            sh.sharded_topk_dev(c, dq[b][name], a.k)
        oi, os_ = sh.sharded_topk_dev(caches["exact"], dq[b]["exact"], a.k)
        torch.cuda.synchronize()
        merged[b] = (oi.cpu().numpy(), os_.cpu().numpy())
        mine = torch.tensor([caches["exact"].exact_stats(b)[4]], dtype=torch.int32, device="cuda")
        every = [torch.zeros_like(mine) for _ in range(world)]
        dist.all_gather(every, mine)
        fallback[b] = [int(x.item()) for x in every]
        for _ in range(a.reps):
            for name, c in caches.items():
                dist.barrier()
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                sh.sharded_topk_dev(c, dq[b][name], a.k)
                torch.cuda.synchronize()
                times[(name, b)].append((time.perf_counter() - t0) * 1e3)
    for c in caches.values():
        c.close()
    if rank == 0:
        whole = pkg.Cache(a.n, a.d, device=local, exact=True, sum_rule=a.rule)
        whole.add(rows)
        equal = {}
        for b, q in queries.items():
            wi, ws = whole.topk(q, a.k)
            mi, ms = merged[b]
            equal[f"b{b}"] = bool(np.array_equal(mi, wi) and np.array_equal(ms.view(np.uint32), ws.view(np.uint32)))
        whole.close()
        print(json.dumps({
            "card": card, "world": world, "n": a.n, "d": a.d, "k": a.k, "rule": a.rule,
            "ms": {f"{name} b{b}": {"median": float(np.median(v)), "min": float(np.min(v)), "max": float(np.max(v))}
                   for (name, b), v in times.items()},
            "exact_fallback_queries_per_rank": {f"b{b}": v for b, v in fallback.items()},
            "exact_merged_equals_unsharded": equal,
        }))
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
