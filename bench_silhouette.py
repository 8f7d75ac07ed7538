"""ClusteringEvaluator's silhouette (b2k_silhouette) per GPU on blobs made as bench.py makes them (k centres ~
U(-10, 10)^d, unit noise, the blob index as the cluster id):

  cfg2       10 M x 128, K = 64     (bench.py's BASELINE cfg2 shape; wgmma pass)
  k1000      10 M x 128, K = 1000   (eight blocks of 128 means per tile; wgmma pass)
  generic    12.5 M x 256, K = 256  (d > 128: the fp64 SIMT pass)

Prints one JSON line: per workload the per-pass device times (CUDA events, option time_kernels: cluster ids, statistics
with its allreduce and the means, the silhouette pass), the bytes of X over each pass's time (TB/s), the useful rate
2 n K d / silhouette pass (TFLOP/s; the wgmma pass issues 3x that in TF32), the whole C-ABI call (host clock around a
synchronised call), a chunked fp64 torch.mm restatement of the same closed form on the device as a baseline and its
difference from the call's value, scikit-learn's silhouette_score on a 20 k-row subsample (CPU seconds, for scale),
and the card's name and power limit.
"""
from __future__ import annotations

import argparse
import json
import subprocess
import time

WORKLOADS = {"cfg2": (10_000_000, 128, 64), "k1000": (10_000_000, 128, 1000), "generic": (12_500_000, 256, 256)}


def card() -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, pl = [s.strip() for s in out.split(",")]
        return {"gpu": name, "power_limit": pl}
    except Exception as e:   # the numbers stand without it, but say so
        return {"gpu": f"unknown ({e})", "power_limit": "unknown"}


def blobs(torch, n, d, k):
    g = torch.Generator(device="cuda").manual_seed(42)
    C = torch.rand((k, d), generator=g, device="cuda") * 20.0 - 10.0
    g = torch.Generator(device="cuda").manual_seed(1234)
    X = torch.empty((n, d), dtype=torch.float32, device="cuda")
    ids = torch.empty((n,), dtype=torch.int64, device="cuda")
    for s in range(0, n, 1_000_000):
        e = min(n, s + 1_000_000)
        z = torch.randint(0, k, (e - s,), generator=g, device="cuda")
        X[s:e] = C[z] + torch.randn((e - s, d), generator=g, device="cuda")
        ids[s:e] = z
    return X, ids


def torch_silhouette(torch, X, ids, k, chunk=262144):
    """The closed form in fp64 with torch on the device: per-cluster sums, then D = ||x'||^2 + ||mu'||^2 - 2 x'.mu'
    + Psi per chunk of rows in the frame of the global mean."""
    n, d = X.shape
    m = X.double().mean(0)
    N = torch.bincount(ids, minlength=k).double()
    S = torch.zeros((k, d), dtype=torch.float64, device=X.device)
    Q = torch.zeros(k, dtype=torch.float64, device=X.device)
    for s in range(0, n, chunk):
        z = X[s:s + chunk].double() - m
        S.index_add_(0, ids[s:s + chunk], z)
        Q.index_add_(0, ids[s:s + chunk], (z * z).sum(1))
    mu = S / N[:, None]
    psi = Q / N - (mu * mu).sum(1)
    mn = (mu * mu).sum(1)
    tot = torch.zeros((), dtype=torch.float64, device=X.device)
    for s in range(0, n, chunk):
        z = X[s:s + chunk].double() - m
        lab = ids[s:s + chunk]
        D = (z * z).sum(1, keepdim=True) + mn[None, :] - 2.0 * torch.mm(z, mu.T) + psi[None, :]
        r = torch.arange(z.shape[0], device=X.device)
        no = N[lab]
        a = D[r, lab].clamp_min(0) * no / (no - 1).clamp_min(1)
        D[r, lab] = float("inf")
        b = D.min(1).values.clamp_min(0)
        sv = torch.where(a < b, 1 - a / b, torch.where(a > b, b / a - 1, torch.zeros_like(a)))
        tot += torch.where(no > 1, sv, torch.zeros_like(sv)).sum()
    return float(tot / n)


def run(torch, ctx, name, steps, warmup):
    n, d, k = WORKLOADS[name]
    X, ids = blobs(torch, n, d, k)
    ctx.set_option("time_kernels", 1)
    for _ in range(warmup):
        ctx.silhouette(X, ids)
    ph = {"ids": 0.0, "stats": 0.0, "silhouette": 0.0, "loop": 0.0}
    walls = []
    for _ in range(steps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        v = ctx.silhouette(X, ids)
        walls.append((time.perf_counter() - t0) * 1e3)
        st = ctx.stats()
        for key, f in (("ids", "last_finalize_ms"), ("stats", "last_reduce_ms"), ("silhouette", "last_fused_ms"),
                       ("loop", "last_loop_ms")):
            ph[key] += st[f] / steps
    path = ctx.stats()["last_path"]
    ctx.set_option("time_kernels", 0)
    xb = n * d * 4
    torch_silhouette(torch, X, ids, k)   # warm-up
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    tv = torch_silhouette(torch, X, ids, k)
    torch.cuda.synchronize()
    torch_ms = (time.perf_counter() - t0) * 1e3
    sk = {}
    try:
        from sklearn.metrics import silhouette_score

        idx = torch.randperm(n, generator=torch.Generator().manual_seed(0))[:20000]
        Xs, ls = X[idx.cuda()].cpu().numpy(), ids[idx.cuda()].cpu().numpy()
        t0 = time.perf_counter()
        silhouette_score(Xs, ls, metric="sqeuclidean")
        sk = {"sklearn_20k_rows_s": round(time.perf_counter() - t0, 3)}
    except Exception as e:   # scikit-learn is optional here
        sk = {"sklearn_20k_rows": f"not run ({e})"}
    del X, ids
    torch.cuda.empty_cache()
    return {"workload": name, "n": n, "d": d, "K": k, "path": "wgmma" if path == 2 else "generic", "value": v,
            "ms": {key: round(val, 3) for key, val in ph.items()}, "call_ms_median": round(sorted(walls)[len(walls) // 2], 3),
            "stats_TBps_of_X": round(xb / (ph["stats"] * 1e-3) / 1e12, 3),
            "silhouette_TBps_of_X": round(xb / (ph["silhouette"] * 1e-3) / 1e12, 3),
            "silhouette_useful_TFLOPs": round(2.0 * n * k * d / (ph["silhouette"] * 1e-3) / 1e12, 1),
            "torch_fp64_ms": round(torch_ms, 2), "torch_value_diff": abs(v - tv), **sk}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    args = ap.parse_args()
    import torch

    from spark_rapids_ml_b200 import _native

    if not torch.cuda.is_available():
        raise SystemExit("bench_silhouette.py needs a CUDA device")
    ctx = _native.Context(0)
    res = [run(torch, ctx, w, args.steps, args.warmup) for w in args.workloads.split(",")]
    ctx.close()
    print(json.dumps({"bench": "silhouette", **card(), "results": res}))


if __name__ == "__main__":
    main()
