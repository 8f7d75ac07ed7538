"""Exact k-NN at BASELINE cfg5's per-GPU shape: 10 M / 8 = 1.25 M items x 100 k queries x d = 128 on one GPU.

Prints one JSON line: per-phase device times of b2k_knn_search (CUDA events, option time_kernels) after warm-up, the
useful rate 2 n_q n_items d / search time, the issued 3xTF32 rate (3x the useful one) as a share of the H100 SXM data-sheet
dense TF32 rate (495 TFLOP/s), the cuBLAS route on the same data (chunked fp32 torch.mm with TF32 off + torch.topk), an
accuracy check of a 1000-query sample against an fp64 restatement on the device, and the card's name and power limit.
k = 5 is the estimator default and k = 64 the largest on the wgmma path; the reference benchmark's default k = 200 takes
the generic path.
"""
from __future__ import annotations

import argparse
import json
import subprocess
import time

import numpy as np

DATASHEET_TF32 = 495e12
TAU_C = 4e-6   # the parity rule's tolerance TAU_C (||q - m||^2 + max ||x - m||^2), m = item mean (tests/knn_oracle.py)


def card() -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, pl = [s.strip() for s in out.split(",")]
        return {"gpu": name, "power_limit": pl}
    except Exception as e:   # the numbers stand without it, but say so
        return {"gpu": f"unknown ({e})", "power_limit": "unknown"}


def torch_route(torch, X, Q, k, chunk=1024):
    xn = (X * X).sum(1)
    D = torch.empty((Q.shape[0], k), dtype=torch.float32, device=X.device)
    I = torch.empty((Q.shape[0], k), dtype=torch.int64, device=X.device)
    for q0 in range(0, Q.shape[0], chunk):
        s = xn[None, :] - 2.0 * torch.mm(Q[q0:q0 + chunk], X.T)
        v, i = torch.topk(s, k, dim=1, largest=False)
        D[q0:q0 + chunk], I[q0:q0 + chunk] = v, i
    return D, I


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--items", type=int, default=1_250_000)
    ap.add_argument("--queries", type=int, default=100_000)
    ap.add_argument("--d", type=int, default=128)
    ap.add_argument("--k", type=int, nargs="+", default=[5, 64])
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--sample", type=int, default=1000)
    args = ap.parse_args()

    import torch

    from spark_rapids_ml_b200 import _native

    if not torch.cuda.is_available():
        raise SystemExit("bench_knn.py measures on a GPU; none is visible")
    torch.backends.cuda.matmul.allow_tf32 = False
    g = torch.Generator(device="cuda").manual_seed(0)
    X = torch.randn((args.items, args.d), generator=g, device="cuda")
    Q = torch.randn((args.queries, args.d), generator=g, device="cuda")
    useful = 2.0 * args.items * args.queries * args.d
    out = {"workload": "exact kNN, BASELINE cfg5 per GPU", "n_items": args.items, "n_queries": args.queries,
           "d": args.d, "steps": args.steps, "results": []}
    with _native.Context(0) as ctx:
        ctx.set_option("time_kernels", 1)
        for k in args.k:
            ph = {"prep": [], "search": [], "merge_refine": [], "allgathers": [], "call": []}
            for it in range(args.warmup + args.steps):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                dist, idx = ctx.knn_search(X, Q, k)
                torch.cuda.synchronize()
                t1 = time.perf_counter()
                st = ctx.stats()
                if it >= args.warmup:
                    ph["prep"].append(st["last_finalize_ms"])
                    ph["search"].append(st["last_fused_ms"])
                    ph["merge_refine"].append(st["last_reduce_ms"])
                    ph["allgathers"].append(st["last_allreduce_ms"])
                    ph["call"].append((t1 - t0) * 1e3)
            path = {2: "wgmma 3xTF32", 1: "generic SIMT"}.get(st["last_path"], str(st["last_path"]))
            search_ms = float(np.median(ph["search"]))
            # cuBLAS route on the same data
            tt = []
            for it in range(args.warmup + args.steps):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                tD, tI = torch_route(torch, X, Q, k)
                torch.cuda.synchronize()
                if it >= args.warmup:
                    tt.append((time.perf_counter() - t0) * 1e3)
            del tD, tI
            # accuracy: a sample of queries against fp64 on the device (parity rule of tests/knn_oracle.py)
            sq = Q[: args.sample].double()
            X64 = X.double()
            xn64 = (X64 * X64).sum(1)
            m = X64.mean(0)
            r2 = float(((X64 - m) ** 2).sum(1).max())
            bad = 0
            for q0 in range(0, sq.shape[0], 100):
                q = sq[q0:q0 + 100]
                d2 = (q * q).sum(1)[:, None] + xn64[None, :] - 2.0 * (q @ X64.T)
                ref = torch.topk(d2, k, dim=1, largest=False).values
                mine = torch.gather(d2, 1, idx[q0:q0 + 100])
                tau = TAU_C * (((q - m) ** 2).sum(1) + r2)
                bad += int(((torch.sort(mine, 1).values - ref).abs() > tau[:, None]).any(1).sum())
            del X64, d2
            res = {"k": k, "path": path,
                   "prep_ms": round(float(np.median(ph["prep"])), 3),
                   "search_ms": round(search_ms, 3),
                   "merge_refine_ms": round(float(np.median(ph["merge_refine"])), 3),
                   "allgathers_ms": round(float(np.median(ph["allgathers"])), 3),
                   "call_ms": round(float(np.median(ph["call"])), 3),
                   "useful_tflops": round(useful / (search_ms * 1e-3) / 1e12, 2),
                   "torch_mm_topk_ms": round(float(np.median(tt)), 3),
                   "speedup_vs_torch_mm": round(float(np.median(tt)) / float(np.median(ph["call"])), 3),
                   "sample_queries_outside_margin": bad, "sample_queries": int(sq.shape[0])}
            if path.startswith("wgmma"):
                res["issued_3xtf32_share_of_datasheet_tf32"] = round(3 * useful / (search_ms * 1e-3) / DATASHEET_TF32, 4)
            out["results"].append(res)
    out.update(card())
    out["note"] = ("k = 200 (the reference benchmark's default) takes the generic SIMT path in this build; "
                   "allgathers are 0 work on one rank")
    print(json.dumps(out))


if __name__ == "__main__":
    main()
