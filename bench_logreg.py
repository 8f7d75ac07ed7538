"""Logistic regression benchmark, per GPU: binomial at 10 M x 128 and 6.25 M x 512, multinomial (K = 10) at 10 M x 128,
float32 rows and labels.

For each shape: the evaluation pass (b2k_logreg_eval on the fused path: margins, residuals and X^T R in one read of X),
timed with CUDA events (option time_kernels) as TB/s of X and fp64 TFLOP/s (4 d K' flops per row); a whole fit at the
default params with a ridge penalty (regParam = 0.01, maxIter 100, tol 1e-6): its time and evaluations; and in the same
run the fp32 torch route on the same device data: one autograd evaluation of the same objective and a
torch.optim.LBFGS fit with the same maxIter (strong-Wolfe line search).  Prints ONE JSON line.

  python bench_logreg.py [--shapes 10000000x128x1,6250000x512x1,10000000x128x10] [--steps 10] [--warmup 2] [--seed 0]

Aims: binomial pass >= 2.3 TB/s; K = 10 pass <= 2 x max(bytes / 3.35 TB/s, flops / 34 TFLOP/s), the data-sheet HBM3
and FP64 (non-tensor) rates of a 700 W H100 SXM.  The card's name and power limit are read in the same run.
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

FP64_TFLOPS = 34.0


def _bench_shape(n: int, d: int, K: int, steps: int, warmup: int, seed: int) -> dict:
    import numpy as np
    import torch

    from spark_rapids_ml_b200 import _native

    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(seed)
    X = torch.randn((n, d), device=dev, generator=g)
    Wt = torch.randn((max(K, 2), d), device=dev, generator=g) / d ** 0.5
    M = X @ Wt.T - torch.log(-torch.log(torch.rand((n, max(K, 2)), device=dev, generator=g)))
    y = (M[:, 0] < M[:, 1]).float() if K == 1 else M.argmax(1).float()
    y = y.contiguous()
    del M
    kp = 1 if K == 1 else K
    classes = np.arange(max(K, 2), dtype=np.float64)
    rng = np.random.default_rng(seed)
    W = rng.normal(size=(kp, d)) * 0.1 / np.sqrt(d)
    b = rng.normal(size=kp) * 0.1
    med = lambda v: statistics.median(v) if v else 0.0  # noqa: E731
    out: dict = {"rows": n, "d": d, "classes": max(K, 2), "margins_per_row": kp}
    bytes_x = 4.0 * n * d + 4.0 * n
    flops = 4.0 * n * d * kp
    with _native.Context(0) as ctx:
        ctx.set_option("time_kernels", 1)
        ts = []
        for i in range(warmup + steps):
            ctx.logreg_eval(X, y, classes, W, b)
            if i >= warmup:
                ts.append(ctx.stats()["last_fused_ms"])
        st = ctx.stats()
        t = med(ts)
        out["eval_path"] = "fused" if st["last_path"] == 2 else "generic"
        out["eval_ms"] = t
        out["eval_tbs"] = bytes_x / (t * 1e-3) / 1e12
        out["eval_fp64_tflops"] = flops / (t * 1e-3) / 1e12
        floor_ms = max(bytes_x / (HBM_TBS * 1e12), flops / (FP64_TFLOPS * 1e12)) * 1e3
        out["eval_floor_ms"] = floor_ms
        if kp == 1:
            out["aim_tbs_2.3_met"] = out["eval_tbs"] >= 2.3
        else:
            out["aim_2x_floor_met"] = t <= 2.0 * floor_ms
        # a whole fit at the default params with a ridge penalty
        classes_d, counts, _ = ctx.logreg_labels(y)
        s = {"reg": 0.01, "l1_ratio": 0.0, "tol": 1e-6, "max_iter": 100, "fit_intercept": True,
             "standardization": True, "family": "auto"}
        ctx.set_option("time_kernels", 0)
        fit_ms, iters = [], 0
        for i in range(1 + 2):
            torch.cuda.synchronize()
            launches0 = ctx.stats()["fused_tc_launches"]
            t0 = time.perf_counter()
            (_, _, iters), = ctx.logreg_fit(X, y, classes_d, counts, [s])
            t1 = time.perf_counter()
            if i > 0:
                fit_ms.append((t1 - t0) * 1e3)
            evals = ctx.stats()["fused_tc_launches"] - launches0
        out["fit_ms"] = med(fit_ms)
        out["fit_iterations"] = iters
        out["fit_evaluations"] = evals

    # the fp32 torch route on the same device data
    # sigma is folded into the weights, as the device fit does: no extra pass over X per evaluation
    Xs = X.std(0, unbiased=True)
    Xs = torch.where(Xs > 0, Xs, torch.ones_like(Xs))
    yi = y.long()

    def objective(V: "torch.Tensor", bb: "torch.Tensor") -> "torch.Tensor":
        Z = X @ (V / Xs).T + bb
        if kp == 1:
            loss = torch.nn.functional.binary_cross_entropy_with_logits(Z[:, 0], y)
        else:
            loss = torch.nn.functional.cross_entropy(Z, yi)
        return loss + 0.5 * 0.01 * (V * V).sum()

    V = torch.zeros((kp, d), device=dev, requires_grad=True)
    bb = torch.zeros((kp,), device=dev, requires_grad=True)
    ev = []
    for i in range(warmup + steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        V.grad = bb.grad = None
        objective(V, bb).backward()
        e1.record()
        torch.cuda.synchronize()
        if i >= warmup:
            ev.append(e0.elapsed_time(e1))
    out["torch_fp32_eval_ms"] = med(ev)
    V = torch.zeros((kp, d), device=dev, requires_grad=True)
    bb = torch.zeros((kp,), device=dev, requires_grad=True)
    opt = torch.optim.LBFGS([V, bb], max_iter=100, history_size=10, tolerance_grad=1e-6, line_search_fn="strong_wolfe")

    def closure() -> "torch.Tensor":
        opt.zero_grad()
        loss = objective(V, bb)
        loss.backward()
        return loss

    torch.cuda.synchronize()
    t0 = time.perf_counter()
    opt.step(closure)
    torch.cuda.synchronize()
    out["torch_fp32_lbfgs_fit_ms"] = (time.perf_counter() - t0) * 1e3
    out["torch_fp32_lbfgs_evaluations"] = int(opt.state[opt._params[0]]["func_evals"])
    del X, y
    torch.cuda.empty_cache()
    return out


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--shapes", default="10000000x128x1,6250000x512x1,10000000x128x10")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_logreg.py needs a CUDA device")
    res = {"card": _card(), "shapes": []}
    for s in a.shapes.split(","):
        n, d, K = (int(v) for v in s.split("x"))
        res["shapes"].append(_bench_shape(n, d, K, a.steps, a.warmup, a.seed))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
