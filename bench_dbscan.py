"""DBSCAN per GPU on blobs, as the reference's benchmark runs it (--eps 100 --min_samples 5 on `blobs`): 1 M x 128 (the
wgmma pass) and 200 k x 256 (the generic pass).

Prints one JSON line: per-phase device times of b2k_dbscan_fit (CUDA events, option time_kernels) after warm-up; the
useful rate 2 n^2 d / pass of the count and union passes and, on the wgmma pass, the issued 3xTF32 rate (3x the useful
one) as a share of the H100 SXM data-sheet dense TF32 rate (495 TFLOP/s); the unions attempted and the pairs decided by
the fp64 rule (option collect_recheck); a baseline count pass (chunked fp32 torch.mm with TF32 off); a check of a
1000-row sample on the device in fp64 (each sampled row is core exactly when its fp64 neighbour count reaches
min_samples, and sampled adjacent core pairs share a label); and the card's name and power limit.
"""
from __future__ import annotations

import argparse
import json
import subprocess
import time

DATASHEET_TF32 = 495e12


def card() -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, pl = [s.strip() for s in out.split(",")]
        return {"gpu": name, "power_limit": pl}
    except Exception as e:   # the numbers stand without it, but say so
        return {"gpu": f"unknown ({e})", "power_limit": "unknown"}


def blobs(torch, n, d, eps, seed, k=1000):
    """k centres uniform in [-1000, 1000]^d (far apart next to eps), rows at std 0.6 eps / sqrt(2 d) around them."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    C = (torch.rand((k, d), generator=g, device="cuda") * 2.0 - 1.0) * 1000.0
    lab = torch.randint(0, k, (n,), generator=g, device="cuda")
    return C[lab] + torch.randn((n, d), generator=g, device="cuda") * (0.6 * eps / (2.0 * d) ** 0.5)


def torch_count(torch, X, eps, chunk=1024):
    """Neighbour counts through chunked fp32 torch.mm (TF32 off): the cuBLAS route to the count pass."""
    xn = (X * X).sum(1)
    cnt = torch.empty(X.shape[0], dtype=torch.int64, device=X.device)
    for i0 in range(0, X.shape[0], chunk):
        D = xn[i0:i0 + chunk, None] + xn[None, :] - 2.0 * torch.mm(X[i0:i0 + chunk], X.T)
        cnt[i0:i0 + chunk] = (D <= eps * eps).sum(1)
    return cnt


def sample_check(torch, X, eps, ms, labels, core, m=1000, seed=0, chunk=65536):
    g = torch.Generator(device="cuda").manual_seed(seed)
    idx = torch.randperm(X.shape[0], generator=g, device="cuda")[:m]
    S = X[idx].double()
    cnt = torch.zeros(m, dtype=torch.int64, device=X.device)
    for j0 in range(0, X.shape[0], chunk):
        Xj = X[j0:j0 + chunk].double()
        D = torch.cdist(S, Xj) ** 2
        cnt += (D <= eps * eps).sum(1)
    core_bad = int(((cnt >= ms) != core[idx]).sum())
    Ds = torch.cdist(S, S) ** 2
    cs = core[idx]
    adj = (Ds <= eps * eps) & cs[:, None] & cs[None, :]
    li = labels[idx].long()
    pair_bad = int((adj & (li[:, None] != li[None, :])).sum())
    return {"sample_rows": m, "core_flag_mismatches": core_bad, "adjacent_core_pairs": int(adj.sum()),
            "adjacent_core_pairs_with_different_labels": pair_bad}


def run(torch, _native, n, d, eps, ms, steps, warmup, path, baseline):
    X = blobs(torch, n, d, eps, seed=d)
    useful = 2.0 * n * n * d
    res = {"n": n, "d": d, "eps": eps, "min_samples": ms}
    with _native.Context(0) as ctx:
        ctx.set_option("time_kernels", 1)
        ctx.set_option("kernel_path", path)
        ph = {"prep": [], "count": [], "union": [], "merge_labels": [], "call": []}
        for it in range(warmup + steps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            labels, core, ncl = ctx.dbscan_fit(X, eps, ms)
            torch.cuda.synchronize()
            t1 = time.perf_counter()
            st = ctx.stats()
            if it >= warmup:
                ph["prep"].append(st["last_finalize_ms"])
                ph["count"].append(st["last_fused_ms"])
                ph["union"].append(st["last_reduce_ms"])
                ph["merge_labels"].append(st["last_allreduce_ms"])
                ph["call"].append((t1 - t0) * 1e3)
        res["path"] = {1: "generic", 2: "wgmma"}[st["last_path"]]
        ctx.set_option("time_kernels", 0)
        ctx.set_option("collect_recheck", 1)
        ctx.dbscan_fit(X, eps, ms)
        st = ctx.stats()
        res["pairs_decided_fp64"] = st["recheck_candidates"]
        res["unions_attempted"] = st["recheck_rows"]
    ms_ = {k: min(v) for k, v in ph.items()}
    res["ms_min"] = {k: round(v, 3) for k, v in ms_.items()}
    res["n_clusters"] = ncl
    res["noise_rows"] = int((labels < 0).sum())
    res["core_rows"] = int(core.sum())
    for p in ("count", "union"):
        res[f"{p}_useful_tflops"] = round(useful / (ms_[p] * 1e-3) / 1e12, 2)
        if res["path"] == "wgmma":
            res[f"{p}_issued_3xtf32_share_of_datasheet"] = round(3 * useful / (ms_[p] * 1e-3) / DATASHEET_TF32, 3)
    res["union_over_count"] = round(ms_["union"] / ms_["count"], 3)
    if baseline:
        torch.backends.cuda.matmul.allow_tf32 = False
        torch_count(torch, X[:4096], eps)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        torch_count(torch, X, eps)
        torch.cuda.synchronize()
        res["torch_mm_count_ms"] = round((time.perf_counter() - t0) * 1e3, 3)
    res["sample_check"] = sample_check(torch, X, eps, ms, labels, core)
    return res


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--eps", type=float, default=100.0)
    ap.add_argument("--min_samples", type=int, default=5)
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--shapes", default="1000000x128,200000x256")
    ap.add_argument("--no-baseline", action="store_true")
    args = ap.parse_args()

    import torch

    from spark_rapids_ml_b200 import _native

    if not torch.cuda.is_available():
        raise SystemExit("bench_dbscan.py measures on a GPU; none is visible")
    out = {"workload": "DBSCAN on blobs per GPU", "steps": args.steps, "results": []}
    for shape in args.shapes.split(","):
        n, d = (int(v) for v in shape.split("x"))
        path = 2 if d % 4 == 0 and 4 <= d <= 128 else 1
        out["results"].append(run(torch, _native, n, d, args.eps, args.min_samples, args.steps, args.warmup, path,
                                  not args.no_baseline))
    out.update(card())
    print(json.dumps(out))


if __name__ == "__main__":
    main()
