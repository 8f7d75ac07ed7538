"""Linear regression benchmark, per GPU: 6.25 M x 512 (BASELINE config 4's shape, so the Gram pass compares with
bench_pca.py) and 10 M x 128, float32 rows and labels.

Times, with CUDA events on the library's stream (option time_kernels): the column-sum pass (X and y), the Gram pass, the
k_xty pass and the two allreduces (0 work on one rank); the host solve for OLS, ridge and the elastic net; the whole fit
(moments + one solve); a 6-setting grid solved from one moments call against 6 separate fits (what fitMultiple does
against per-map fits); and the prediction kernel.  In the same run, the route a cuBLAS-backed implementation takes:
torch.mm(Xc^T, [Xc | yc]) in fp32 with TF32 disabled on the centred data, then an fp64 solve on the host.  Both moment
matrices are compared with an fp64 restatement formed on the device in chunks.  Prints ONE JSON line.

  python bench_linreg.py [--gpus 1] [--shapes 6250000x512,10000000x128] [--steps 5] [--warmup 2] [--seed 0]

Rates: pass GB/s = bytes the pass must read (4 n d for X, + 4 n for y) over its time; predict GB/s = (4 n d + 8 n)
bytes over its kernel time; each against the 3.35 TB/s HBM3 data-sheet figure.  The aims: k_xty within 1.25x of the
column-sum pass on X, predict >= 2.3 TB/s.  The card's name and power limit are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_pca import HBM_TBS, _card  # noqa: E402

GRID = [(0.0, 0.0), (0.1, 0.0), (1.0, 0.0), (0.05, 1.0), (0.05, 0.5), (0.2, 0.5)]   # (regParam, elasticNetParam)


def _bench_shape(n: int, d: int, steps: int, warmup: int, seed: int) -> dict:
    import numpy as np
    import torch

    from spark_rapids_ml_b200 import _native

    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(seed)
    X = torch.randn((n, d), device=dev, generator=g) + 3.0
    w_true = torch.randn((d,), device=dev, generator=g) / d ** 0.5
    y = (X @ w_true + 0.5 * torch.randn((n,), device=dev, generator=g) + 1.0).float().contiguous()
    ev = lambda: torch.cuda.Event(enable_timing=True)  # noqa: E731
    med = lambda v: statistics.median(v) if v else 0.0  # noqa: E731
    out: dict = {"rows": n, "d": d}

    # fp64 restatement of the moments, on the device in chunks
    mu = torch.cat([X.sum(0, dtype=torch.float64), y.sum(dtype=torch.float64)[None]]) / n
    M_ref = torch.zeros((d + 1, d + 1), dtype=torch.float64, device=dev)
    for r in range(0, n, 1 << 18):
        V = torch.cat([X[r:r + (1 << 18)].double(), y[r:r + (1 << 18), None].double()], 1) - mu
        M_ref += V.T @ V
        del V
    M_ref = M_ref.cpu().numpy()
    scale = float(np.abs(M_ref).max())

    with _native.Context(0) as ctx:
        ctx.set_option("time_kernels", 1)
        ph = {"colsum_ms": [], "gram_ms": [], "xty_ms": [], "allreduce_ms": [], "moments_ms": [], "fit_ms": []}
        for i in range(warmup + steps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            nt, mean, mom = ctx.linreg_moments(X, y)
            _native.linreg_solve(mean, mom, nt, 0.1, 0.0)
            t1 = time.perf_counter()
            if i >= warmup:
                st = ctx.stats()
                ph["colsum_ms"].append(st["last_reduce_ms"])
                ph["gram_ms"].append(st["last_fused_ms"])
                ph["xty_ms"].append(st["last_finalize_ms"])
                ph["allreduce_ms"].append(st["last_allreduce_ms"])
                ph["moments_ms"].append(st["last_loop_ms"])
                ph["fit_ms"].append((t1 - t0) * 1e3)
        out.update({k: round(med(v), 3) for k, v in ph.items()})
        out["gram_path"] = "wgmma" if ctx.stats()["last_path"] == 2 else "generic"
        out["moments_max_dev_rel"] = float(np.abs(mom - M_ref).max() / scale)
        for name, (reg, l1) in (("ols", (0.0, 0.0)), ("ridge", (0.1, 0.0)), ("elastic_net", (0.05, 0.5))):
            ts = []
            for _ in range(3):
                t0 = time.perf_counter()
                _native.linreg_solve(mean, mom, nt, reg, l1)
                ts.append((time.perf_counter() - t0) * 1e3)
            out[f"solve_{name}_ms"] = round(med(ts), 3)

        # 6-setting grid: one moments call + 6 solves, against 6 x (moments + solve)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        nt, mean, mom = ctx.linreg_moments(X, y)
        for reg, l1 in GRID:
            _native.linreg_solve(mean, mom, nt, reg, l1)
        out["grid6_one_pass_ms"] = round((time.perf_counter() - t0) * 1e3, 3)
        t0 = time.perf_counter()
        for reg, l1 in GRID:
            nt, mean, mom = ctx.linreg_moments(X, y)
            _native.linreg_solve(mean, mom, nt, reg, l1)
        out["grid6_six_fits_ms"] = round((time.perf_counter() - t0) * 1e3, 3)

        # prediction kernel
        coef, b, _ = _native.linreg_solve(mean, mom, nt, 0.1, 0.0)
        w = torch.from_numpy(coef).to(dev)
        for _ in range(warmup):
            ctx.linreg_predict(X, w, b)
        ts = []
        for _ in range(steps):
            e0, e1 = ev(), ev()
            e0.record()
            ctx.linreg_predict(X, w, b)
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1))
        out["predict_ms"] = round(med(ts), 3)
        pred = ctx.linreg_predict(X[:100000], w, b).cpu().numpy()
        ref = b + X[:100000].double().cpu().numpy() @ coef
        out["predict_max_dev_rel"] = float(np.abs(pred - ref).max() / np.abs(ref).max())

    # the cuBLAS route: fp32 torch.mm of Xc^T [Xc | yc], TF32 off, then an fp64 solve on the host
    torch.backends.cuda.matmul.allow_tf32 = False
    V = torch.empty((n, d + 1), dtype=torch.float32, device=dev)
    ts = []
    for i in range(warmup + steps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        mu32 = torch.cat([X.mean(0, dtype=torch.float64), y.mean(dtype=torch.float64)[None]]).float()
        V[:, :d] = X - mu32[:d]
        V[:, d] = y - mu32[d]
        Mb = torch.mm(V[:, :d].T, V).double().cpu().numpy()
        Mb = np.vstack([Mb, np.r_[Mb[:, d], (V[:, d].double() @ V[:, d].double()).item()]])
        _native.linreg_solve(mu.cpu().numpy(), Mb, n, 0.1, 0.0)
        if i >= warmup:
            ts.append((time.perf_counter() - t0) * 1e3)
    out["torch_mm_route_ms"] = round(med(ts), 3)
    out["torch_mm_max_dev_rel"] = float(np.abs(Mb - M_ref).max() / scale)
    del V

    gb = 1e-9
    out["colsum_gbs"] = round((4 * n * d + 4 * n) * gb / (out["colsum_ms"] * 1e-3), 1) if out["colsum_ms"] else None
    out["xty_gbs"] = round((4 * n * d + 4 * n) * gb / (out["xty_ms"] * 1e-3), 1) if out["xty_ms"] else None
    out["xty_over_colsum"] = round(out["xty_ms"] / out["colsum_ms"], 3) if out["colsum_ms"] else None
    out["xty_aim_met"] = bool(out["xty_over_colsum"] is not None and out["xty_over_colsum"] <= 1.25)
    out["predict_gbs"] = round((4 * n * d + 8 * n) * gb / (out["predict_ms"] * 1e-3), 1)
    out["predict_share_of_hbm"] = round(out["predict_gbs"] / (HBM_TBS * 1e3), 3)
    out["predict_aim_met"] = bool(out["predict_gbs"] >= 2300.0)
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--shapes", default="6250000x512,10000000x128")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args()
    if a.gpus != 1:
        raise SystemExit("bench_linreg.py measures one GPU; --gpus must be 1")
    import torch

    assert torch.cuda.is_available(), "bench_linreg.py needs a CUDA device"
    res = {"bench": "linreg", **_card(), "shapes": []}
    for s in a.shapes.split(","):
        n, d = (int(v) for v in s.lower().split("x"))
        res["shapes"].append(_bench_shape(n, d, a.steps, a.warmup, a.seed))
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
