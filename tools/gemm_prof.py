"""Times the four projection GEMMs of one ModernBERT-base layer in the configuration the encoder runs them in, at
T = M tokens (default 131072 = the headline batch 256 x seq 512):

  Wqkv  EPI_ROPE,     LayerNorm-fold consumer (fold stats, RoPE on the q/k columns)   N = 2304, K = 768
  Wo    EPI_RESID_HL, fp16-pair residual producer (row stats, pivots in and out)      N = 768,  K = 768
  Wi    EPI_GEGLU,    LayerNorm-fold consumer                                         N = 2304, K = 768
  Wo2   EPI_RESID_HL                                                                  N = 768,  K = 1152

Per GEMM: CUDA-event time over many launches, TFLOP/s, the algorithmic HBM bytes over that time, the modelled
L2 -> SM operand traffic over that time for the thread-block cluster the library launches (each of the cluster_n CTAs
loads 1/cluster_n of the shared A box and multicasts it to the others; W boxes are loaded per CTA), the number of
co-resident clusters (workers of the persistent grid), and torch.mm on the same fp16 M, N, K as a cuBLAS reference point (no epilogue: a
reference, not a target).  The GPU name, power limit and maximum SM clock are read in the same run.

  python tools/gemm_prof.py [--root TREE] [--iters N] [--json OUT] [--only Wqkv,Wi]

--root loads the library built in another checkout of this project (to compare two builds in one run).
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ap = argparse.ArgumentParser()
ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
ap.add_argument("--m", type=int, default=131072)
ap.add_argument("--iters", type=int, default=20)
ap.add_argument("--json", default=None, help="also write the rows as JSON here")
ap.add_argument("--only", default=None, help="comma-separated GEMM names to time")
args = ap.parse_args()
sys.path.insert(0, os.path.abspath(args.root))

import torch  # noqa: E402

import semantic_router_b200 as pkg  # noqa: E402

if not torch.cuda.is_available():
    raise SystemExit("gemm_prof.py: no CUDA device")
H = pkg.hooks()
EPI_ROPE, EPI_GEGLU, EPI_RESID_HL = 1, 3, 6
M, Hd, I = args.m, 768, 1152
dev = "cuda"


def cluster_shape(epi, n, k):
    """(cluster_n, workers) the library launches for this GEMM; a build without clusters has one worker per SM."""
    f = getattr(H, "sr_test_gemm_cluster", None)
    if f is None:
        return 1, torch.cuda.get_device_properties(0).multi_processor_count
    f.argtypes = [C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    cn, w = C.c_int(0), C.c_int(0)
    assert f(epi, n, k, C.byref(cn), C.byref(w)) == 0
    return cn.value, w.value


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                            "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return r.stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f"nvidia-smi unavailable ({e})"


def timed(fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


g = torch.Generator(device=dev).manual_seed(0)
x_h = torch.randn(M, Hd, device=dev, generator=g).half()          # LayerNorm-fold A operand (raw fp16 rows)
x_i = torch.randn(M, I, device=dev, generator=g).half()           # GeGLU output, the Wo2 A operand
fold_stats = torch.rand(Hd // 128, M, 2, device=dev, generator=g) + 1.0
pos = (torch.arange(M, device=dev, dtype=torch.int32) % 512).contiguous()
cos = torch.rand(1024, 32, device=dev, generator=g)
sin = torch.rand(1024, 32, device=dev, generator=g)
w_qkv = (torch.randn(3 * Hd, Hd, device=dev, generator=g) * 0.02).half()
w_i = (torch.randn(2 * I, Hd, device=dev, generator=g) * 0.02).half()
w_o = (torch.randn(Hd, Hd, device=dev, generator=g) * 0.02).half()
w_o2 = (torch.randn(Hd, I, device=dev, generator=g) * 0.02).half()
qkv = torch.empty(M, 3 * Hd, device=dev, dtype=torch.float16)
mid = torch.empty(M, I, device=dev, dtype=torch.float16)
hi = torch.randn(M, Hd, device=dev, generator=g).half()
lo = torch.zeros(M, Hd, device=dev, dtype=torch.float16)
parts = Hd // 128
recs = [torch.zeros(parts * M * 2 + M, device=dev) for _ in range(2)]   # [row stats | pivots], alternating in / out
flip = [0]


def p(t):
    return t.data_ptr()


def call_fold(a, w, out, n, epi, n_out, rope_cols):
    rope = dict(pos=pos, rope_cos=cos, rope_sin=sin, rope_cols=rope_cols) if epi == EPI_ROPE else {}
    rc, _ = pkg.binding.run_gemm(m=M, n=n, k=Hd, a=a, w=w, out=out, ldo=n_out, epi=epi, fold_stats=fold_stats,
                                 fold_eps=1e-5, fold_h=Hd, **rope)
    assert rc == 0


def call_resid_hl(a, w, k):
    dst, prev = recs[flip[0]], recs[flip[0] ^ 1]
    flip[0] ^= 1
    rc = H.sr_test_gemm_resid_hl(p(a), p(w), p(hi), p(lo), M, Hd, k, None, p(dst), dst[parts * M * 2:].data_ptr(),
                                 prev[parts * M * 2:].data_ptr(), p(prev))
    assert rc == 0


# (name, epilogue, N, K, launch, HBM bytes: A + outputs (+ residual pair read) + row statistics)
gemms = [
    ("Wqkv", "EPI_ROPE fold", EPI_ROPE, 3 * Hd, Hd, lambda: call_fold(x_h, w_qkv, qkv, 3 * Hd, EPI_ROPE, 3 * Hd, 2 * Hd),
     M * Hd * 2 + M * 3 * Hd * 2 + parts * M * 8 + 3 * Hd * Hd * 2),
    ("Wo", "EPI_RESID_HL", EPI_RESID_HL, Hd, Hd, lambda: call_resid_hl(x_h, w_o, Hd),
     M * Hd * 2 + 4 * M * Hd * 2 + 2 * parts * M * 8 + Hd * Hd * 2),
    ("Wi", "EPI_GEGLU fold", EPI_GEGLU, 2 * I, Hd, lambda: call_fold(x_h, w_i, mid, 2 * I, EPI_GEGLU, I, 0),
     M * Hd * 2 + M * I * 2 + parts * M * 8 + 2 * I * Hd * 2),
    ("Wo2", "EPI_RESID_HL", EPI_RESID_HL, Hd, I, lambda: call_resid_hl(x_i, w_o2, I),
     M * I * 2 + 4 * M * Hd * 2 + 2 * parts * M * 8 + Hd * I * 2),
]
BM = BN = 128
info = gpu_info()
print(f"# {info}   M={M}   root={os.path.abspath(args.root)}")
print(f"# {'gemm':5s} {'epilogue':15s} {'N':>5s} {'K':>5s} {'cluster':>7s} {'workers':>7s} {'ms':>7s} {'TFLOP/s':>8s} {'HBM GB/s':>9s} "
      f"{'L2->SM GB/s':>11s} {'mm ms':>7s} {'mm TFLOP/s':>10s}")
rows = []
if args.only:
    gemms = [g_ for g_ in gemms if g_[0] in args.only.split(",")]
for name, epi_name, epi, n, k, fn, hbm in gemms:
    ms = timed(fn, args.iters)
    cn, workers = cluster_shape(epi, n, k)
    # tile width of the kernel this GEMM runs on: 192 for the LayerNorm-fold projections (gemm_wide_kernel)
    bn = 192 if epi in (EPI_ROPE, EPI_GEGLU) else BN
    tiles = ((M + BM - 1) // BM) * ((n + bn - 1) // bn)
    l2_bytes = tiles * k * 2 * (BM / cn + bn)
    a = x_i if k == I else x_h
    w = {"Wqkv": w_qkv, "Wo": w_o, "Wi": w_i, "Wo2": w_o2}[name]
    ms_mm = timed(lambda: torch.mm(a, w.t()), args.iters)
    flops = 2.0 * M * n * k
    row = {"gemm": name, "epilogue": epi_name, "M": M, "N": n, "K": k, "cluster": f"1x{cn}", "clusters": workers, "ms": ms,
           "tflops": flops / ms / 1e9, "hbm_gbs": hbm / ms / 1e6, "l2_sm_gbs": l2_bytes / ms / 1e6, "mm_ms": ms_mm,
           "mm_tflops": flops / ms_mm / 1e9}
    rows.append(row)
    print(f"  {name:5s} {epi_name:15s} {n:5d} {k:5d} {row['cluster']:>7s} {workers:7d} {ms:7.3f} {row['tflops']:8.1f} "
          f"{row['hbm_gbs']:9.0f} {row['l2_sm_gbs']:11.0f} {ms_mm:7.3f} {row['mm_tflops']:10.1f}")
tot = sum(r["ms"] for r in rows)
print(f"# four GEMMs: {tot:.3f} ms per layer, {22 * tot:.1f} ms per 22-layer step")
if args.json:
    os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
    json.dump({"gpu": info, "rows": rows, "layer_ms": tot}, open(args.json, "w"), indent=1)
