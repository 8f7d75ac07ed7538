"""PCA benchmark: BASELINE config 4 per GPU (the 50 M x 512 float32 rows over 8 GPUs = 6.25 M rows each), k = 32.

Times, with CUDA events on the library's stream (option time_kernels): the column-sum pass, the Gram pass, the two
allreduces (0 work on one rank) and the host eigen step; end-to-end fit and transform; and, in the same run, the route a
cuBLAS-backed implementation takes for the Gram matrix: torch.mm(Xc^T, Xc) in fp32 with TF32 disabled on the same centred
matrix.  Both Gram results are compared with an fp64 Gram formed on the device in chunks.  Prints ONE JSON line.

  python bench_pca.py [--gpus 1] [--rows 6250000] [--d 512] [--k 32] [--steps 5] [--warmup 2] [--seed 0]

Rates: useful Gram flops n d (d + 1) (the upper triangle); issued tf32 flops 3 x (computed 128 x 128 block tiles) x
2 x 128 x 128 x n (3xTF32); the share of the 495 TFLOP/s dense-TF32 data-sheet figure (700 W) is issued flops over the
Gram-pass time; pass-1 GB/s is 4 n d bytes over the column-sum time, against 3.35 TB/s.  The card's name and power limit
are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

TF32_DENSE_TFLOPS = 495.0
HBM_TBS = 3.35


def _card() -> dict:
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clk = [x.strip() for x in q.split(",")]
        return {"gpu": name, "power_limit": power, "max_sm_clock": clk}
    except Exception as e:   # the numbers still stand; the card is then named by torch only
        import torch

        return {"gpu": torch.cuda.get_device_name(0), "power_limit": f"unknown ({e.__class__.__name__})"}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--rows", type=int, default=6_250_000)
    ap.add_argument("--d", type=int, default=512)
    ap.add_argument("--k", type=int, default=32)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args()
    if a.gpus != 1:
        raise SystemExit("bench_pca.py measures one GPU (the per-GPU share of config 4); --gpus must be 1")

    import numpy as np
    import torch

    from spark_rapids_ml_b200 import _native

    assert torch.cuda.is_available(), "bench_pca.py needs a CUDA device"
    n, d, k = a.rows, a.d, a.k
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(a.seed)
    scale = 1.0 / torch.sqrt(1.0 + torch.arange(d, device=dev, dtype=torch.float32))
    X = torch.randn((n, d), device=dev, generator=g) * scale + 3.0
    ev = lambda: torch.cuda.Event(enable_timing=True)  # noqa: E731

    with _native.Context(0) as ctx:
        ctx.set_option("time_kernels", 1)
        phases = {"mean_pass_ms": [], "gram_pass_ms": [], "allreduce_ms": [], "eigen_ms": [], "fit_ms": []}
        for i in range(a.warmup + a.steps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = ctx.pca_fit(X, k)   # synchronises its stream before returning
            t1 = time.perf_counter()
            if i >= a.warmup:
                st = ctx.stats()
                phases["mean_pass_ms"].append(st["last_reduce_ms"])
                phases["gram_pass_ms"].append(st["last_fused_ms"])
                phases["allreduce_ms"].append(st["last_allreduce_ms"])
                phases["eigen_ms"].append(st["last_finalize_ms"])
                phases["fit_ms"].append((t1 - t0) * 1e3)
        path = ctx.stats()["last_path"]
        C = torch.from_numpy(out["components_"].astype(np.float32)).to(dev)
        tr = []
        for i in range(a.warmup + a.steps):
            e0, e1 = ev(), ev()
            e0.record()
            Y = ctx.pca_transform(X, C)
            e1.record()
            torch.cuda.synchronize()
            if i >= a.warmup:
                tr.append(e0.elapsed_time(e1))
        del Y
        full = ctx.pca_fit(X, d)   # k = d: the device covariance, reconstructed from its full eigendecomposition
    med = {key: statistics.median(v) for key, v in phases.items()}

    # the library route: fp32 GEMM (no TF32) on the centred matrix, timed with events in the same run
    mu = X.sum(0, dtype=torch.float64) / n
    Xc = X - mu.float()
    del X
    torch.backends.cuda.matmul.allow_tf32 = False
    mm = []
    for i in range(a.warmup + a.steps):
        e0, e1 = ev(), ev()
        e0.record()
        Gt = torch.mm(Xc.T, Xc)
        e1.record()
        torch.cuda.synchronize()
        if i >= a.warmup:
            mm.append(e0.elapsed_time(e1))
    G64 = torch.zeros((d, d), dtype=torch.float64, device=dev)
    for r in range(0, n, 1 << 18):
        xc = Xc[r:r + (1 << 18)].double()
        G64 += xc.T @ xc
    # Xc is centred on fl32(mu); the fp64 Gram of the data centred on mu removes that offset exactly
    delta = (mu - mu.float().double())
    G64 -= n * torch.outer(delta, delta)
    Gt = Gt.double() - n * torch.outer(delta, delta)
    cov64 = (G64 / (n - 1)).cpu().numpy()
    lam = full["singular_values_"] ** 2 / (n - 1)
    cov_dev = full["components_"].T @ np.diag(lam) @ full["components_"]
    scale_c = float(np.abs(cov64).max())
    err_dev = float(np.abs(cov_dev - cov64).max() / scale_c)
    err_mm = float(np.abs((Gt / (n - 1)).cpu().numpy() - cov64).max() / scale_c)

    nblk = (d + 127) // 128
    ntile = nblk * (nblk + 1) // 2
    useful = float(n) * d * (d + 1)
    issued = 3.0 * ntile * 2.0 * 128 * 128 * n
    gram_s = med["gram_pass_ms"] / 1e3
    res = {
        "workload": f"PCA config 4 per GPU: n={n} d={d} k={k} float32",
        "gram_path": {2: "wgmma 3xTF32", 1: "generic SIMT fp64"}.get(path, str(path)),
        "samples_per_s_fit": n / (med["fit_ms"] / 1e3),
        **{key: round(v, 3) for key, v in med.items()},
        "transform_ms": round(statistics.median(tr), 3),
        "transform_hbm_gbs": round((4.0 * n * d + 4.0 * n * k) / (statistics.median(tr) / 1e3) / 1e9, 1),
        "gram_useful_tflops": round(useful / gram_s / 1e12, 1),
        "gram_issued_tf32_tflops": round(issued / gram_s / 1e12, 1),
        "gram_share_of_tf32_datasheet": round(issued / gram_s / 1e12 / TF32_DENSE_TFLOPS, 3),
        "mean_pass_hbm_gbs": round(4.0 * n * d / (med["mean_pass_ms"] / 1e3) / 1e9, 1),
        "mean_pass_share_of_hbm": round(4.0 * n * d / (med["mean_pass_ms"] / 1e3) / 1e12 / HBM_TBS, 3),
        "torch_mm_fp32_gram_ms": round(statistics.median(mm), 3),
        "gram_speedup_vs_torch_mm": round(statistics.median(mm) / med["gram_pass_ms"], 2),
        "cov_max_err_rel_device": err_dev,
        "cov_max_err_rel_torch_mm_fp32": err_mm,
        "steps": a.steps,
        "warmup": a.warmup,
        **_card(),
    }
    print(json.dumps(res))


if __name__ == "__main__":
    main()
