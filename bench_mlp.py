"""Multilayer perceptron benchmark: b2k_mlp_eval / b2k_mlp_fit on seeded data, one GPU, at 10 M x 128 with layers
[128, 64, 32, 10] and 2 M x 784 with layers [784, 128, 10].  Prints one JSON record with, per shape: one evaluation's
device time split per pass (torch.profiler over the library's kernels: row products, cross-Gram, the rest); the
achieved TFLOP/s against the 3xTF32 bound (NVIDIA's H100 SXM data sheet: TF32 495 TFLOP/s, divided by 3) and the time
bound of reading X once from HBM (3.35 TB/s); the fit time at maxIter 100 (L-BFGS); the time of one fp32 torch autograd
loss-and-gradient step on the same data and network; and the card's name and power limit read in the same run.

    python bench_mlp.py [--shapes 10000000:128,64,32,10;2000000:784,128,10] [--max-iter 100]
"""
import argparse
import json
import subprocess
import time

import numpy as np
import torch

from spark_rapids_ml_b200 import _native

HBM = 3.35e12
TF32_3X = 495e12 / 3


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"unavailable: {e}"


def data(n, layers, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    d, C = layers[0], layers[-1]
    R = torch.randn(d, C, device="cuda", generator=g)
    X = torch.empty(n, d, device="cuda", dtype=torch.float32)
    y = torch.empty(n, device="cuda", dtype=torch.float32)
    for s in range(0, n, 1 << 20):
        e = min(n, s + (1 << 20))
        X[s:e] = torch.randn(e - s, d, device="cuda", generator=g)
        y[s:e] = torch.argmax(X[s:e] @ R, dim=1).float()
    return X, y


def flops_per_row(layers):
    """Forward products, backward delta products and the cross-Gram (with its bias column)."""
    L = len(layers) - 1
    fwd = sum(2 * layers[i - 1] * layers[i] for i in range(1, L + 1))
    bwd = sum(2 * layers[i] * layers[i - 1] for i in range(2, L + 1))
    gram = sum(2 * (layers[i - 1] + 1) * layers[i] for i in range(1, L + 1))
    return fwd + bwd + gram


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return r, time.perf_counter() - t0


def pass_split(ctx, X, y, layers, w):
    """Device ms of one evaluation per kernel family (torch.profiler, CUDA activities)."""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        ctx.mlp_eval(X, y, layers, w)
        torch.cuda.synchronize()
    out = {"row_products_ms": 0.0, "cross_gram_ms": 0.0, "other_ms": 0.0, "kernels": []}
    for ev in prof.key_averages():
        name, us = ev.key, ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
        if "k_mlp" not in name:
            continue
        out["kernels"].append([name[name.find("k_mlp"):][:40], ev.count, round(us / 1e3, 3)])
        if "k_mlp_wg" in name and "true>" in name:
            out["cross_gram_ms"] += us / 1e3
        elif "k_mlp_wg" in name:
            out["row_products_ms"] += us / 1e3
        else:
            out["other_ms"] += us / 1e3
    return out


def torch_step_ms(X, y, layers, reps=3):
    """One fp32 autograd loss-and-gradient step over the whole data (the sigmoid network, mean cross-entropy)."""
    mods = []
    for i in range(1, len(layers)):
        mods.append(torch.nn.Linear(layers[i - 1], layers[i]))
        if i < len(layers) - 1:
            mods.append(torch.nn.Sigmoid())
    net = torch.nn.Sequential(*mods).cuda()
    yl = y.long()

    def step():
        net.zero_grad(set_to_none=True)
        loss = torch.nn.functional.cross_entropy(net(X), yl)
        loss.backward()
        return loss

    step()
    ts = [timed(step)[1] for _ in range(reps)]
    return 1e3 * min(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="10000000:128,64,32,10;2000000:784,128,10")
    ap.add_argument("--max-iter", type=int, default=100)
    ap.add_argument("--evals", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_mlp.py needs a GPU")
    torch.backends.cuda.matmul.allow_tf32 = False
    ctx = _native.Context(0)
    res = {"bench": "mlp", "card": card(), "max_iter": a.max_iter, "runs": []}
    for spec in a.shapes.split(";"):
        n_s, lay_s = spec.split(":")
        n, layers = int(n_s), [int(v) for v in lay_s.split(",")]
        X, y = data(n, layers, seed=0)
        P = sum(layers[i] * (layers[i - 1] + 1) for i in range(1, len(layers)))
        w = np.random.default_rng(1).normal(size=P) * 0.3
        ctx.mlp_eval(X[: 1 << 16].contiguous(), y[: 1 << 16].contiguous(), layers, w)   # warm-up
        ctx.mlp_eval(X, y, layers, w)
        ctx.set_option("time_kernels", 1)
        dev = []
        walls = []
        for _ in range(a.evals):
            _, t = timed(lambda: ctx.mlp_eval(X, y, layers, w))
            walls.append(t)
            dev.append(ctx.stats()["last_fused_ms"])
        ctx.set_option("time_kernels", 0)
        eval_ms = float(np.median(dev))
        flops = flops_per_row(layers) * n
        split = pass_split(ctx, X, y, layers, w)
        _, fit_s = timed(lambda: ctx.mlp_fit(X, y, layers, max_iter=a.max_iter, tol=0.0, seed=3))
        fit_stats = ctx.stats()
        tstep = torch_step_ms(X, y, layers)
        bound_ms = 1e3 * max(flops / TF32_3X, n * layers[0] * 4 / HBM)
        res["runs"].append({
            "n": n, "layers": layers, "eval_device_ms": eval_ms, "eval_wall_ms": 1e3 * float(np.median(walls)),
            "pass_split": split, "tflop_per_eval": flops / 1e12, "tflops": flops / (eval_ms / 1e3) / 1e12,
            "share_of_3xtf32_bound": flops / TF32_3X / (eval_ms / 1e3),
            "hbm_bound_ms": 1e3 * n * layers[0] * 4 / HBM, "compute_bound_ms": 1e3 * flops / TF32_3X,
            "eval_over_bound": eval_ms / bound_ms,
            "fit_s": fit_s, "fit_iterations": int(fit_stats["last_n_iter"]), "fit_path": int(fit_stats["last_path"]),
            "torch_fp32_step_ms": tstep, "eval_speedup_vs_torch": tstep / eval_ms,
        })
        del X, y
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
