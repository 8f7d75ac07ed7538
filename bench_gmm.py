"""Gaussian mixture benchmark: b2k_gmm_fit on a seeded 16-component anisotropic mixture at 10 M x 128 (the wgmma E pass)
and a d = 256 case (the generic E pass), one GPU.  Prints one JSON record: per iteration the E, M, host and allreduce
times, each device pass's useful TFLOP/s and share of the 3xTF32 bound (495 / 3 TFLOP/s, NVIDIA's dense TF32 figure for
the H100 SXM), the agreement of the two E paths from the same injected start, an fp32 torch E+M step for comparison,
and the card's name and power limit read in the same run.

    python bench_gmm.py [--n 10000000] [--d 128] [--k 16] [--iters 5]
"""
import argparse
import json
import subprocess
import time

import numpy as np
import torch

from spark_rapids_ml_b200 import _native

TF32_3X = 495e12 / 3


def mixture(n, d, k, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    means = torch.randn(k, d, device="cuda", generator=g, dtype=torch.float64) * 4
    scale = torch.rand(k, d, device="cuda", generator=g, dtype=torch.float64) + 0.5
    z = torch.randint(0, k, (n,), device="cuda", generator=g)
    X = torch.empty(n, d, device="cuda", dtype=torch.float32)
    for s in range(0, n, 1 << 20):
        e = min(n, s + (1 << 20))
        zz = z[s:e]
        # scaled by 1 / 50: MLlib's E-step adds EPS = 2.2e-16 to w pdf, so at d = 128 the densities must exceed it
        # (variances well below 1), or every responsibility is 1 / k and EM stops after two iterations
        X[s:e] = ((means[zz] + torch.randn(e - s, d, device="cuda", generator=g, dtype=torch.float64) * scale[zz])
                  / 50).float()
    return X


def near_start(X, k):
    """k rows spread over the data as means, the data's diagonal variance as every covariance."""
    idx = torch.linspace(0, X.shape[0] - 1, k, device="cuda").long()
    var = X[: 1 << 20].double().var(0).cpu().numpy()
    return np.full(k, 1.0 / k), X[idx].double().cpu().numpy(), np.stack([np.diag(var)] * k)


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"unavailable: {e}"


def run(ctx, X, k, iters, path, init):
    ctx.set_option("kernel_path", path)
    ctx.set_option("time_kernels", 1)
    ctx.gmm_fit(X, k, init=init, max_iter=1, tol=0.0)   # warm-up
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = ctx.gmm_fit(X, k, init=init, max_iter=iters, tol=0.0)
    wall = time.perf_counter() - t0
    st = ctx.stats()
    n, d = X.shape
    e_flop, m_flop = 2.0 * k * d * d * n, 1.0 * k * d * (d + 1) * n
    it = max(out["n_iter"], 1)
    e_ms, m_ms = st["last_fused_ms"] / it, st["last_reduce_ms"] / it
    return out, {"path": "wgmma" if st["last_path"] == _native.PATH_FUSED else "generic", "n": n, "d": d, "k": k,
                 "iters": out["n_iter"], "e_ms": e_ms, "m_ms": m_ms, "host_ms": st["last_finalize_ms"] / it,
                 "allreduce_ms": st["last_allreduce_ms"] / it, "call_s": wall,
                 "e_tflops": e_flop / e_ms / 1e9, "e_share_of_3xtf32": e_flop / TF32_3X / (e_ms / 1e3),
                 "m_tflops": m_flop / m_ms / 1e9, "m_share_of_3xtf32": m_flop / TF32_3X / (m_ms / 1e3)}


def torch_step_ms(X, w, mu, cov, reps=3):
    """One fp32 EM iteration in torch (Cholesky whitening, log-sum-exp, weighted moments), for comparison."""
    Xt = X
    W = torch.tensor(w, device="cuda", dtype=torch.float32)
    M = torch.tensor(mu, device="cuda", dtype=torch.float32)
    C = torch.tensor(cov, device="cuda", dtype=torch.float32)

    def step():
        L = torch.linalg.cholesky(C)
        Li = torch.linalg.inv(L)
        q = torch.stack([((Xt - M[j]) @ Li[j].T).square().sum(1) for j in range(len(w))], 1)
        logp = torch.log(W) - 0.5 * q - torch.log(torch.diagonal(L, dim1=1, dim2=2)).sum(1)
        r = torch.softmax(logp, 1)
        N = r.sum(0)
        mu2 = (r.T @ Xt) / N[:, None]
        cov2 = torch.stack([((Xt - mu2[j]) * r[:, j:j + 1]).T @ (Xt - mu2[j]) / N[j] for j in range(len(w))])
        return cov2

    step()
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    for _ in range(reps):
        step()
    ev[1].record()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1]) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--d", type=int, default=128)
    ap.add_argument("--k", type=int, default=16)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--n-generic", type=int, default=1_000_000)
    a = ap.parse_args()
    rec = {"card": card()}
    with _native.Context(0) as ctx:
        X = mixture(a.n, a.d, a.k, 1)
        init = near_start(X, a.k)
        wg, rec["wgmma"] = run(ctx, X, a.k, a.iters, _native.PATH_AUTO, init)
        Xs = X[: a.n_generic].contiguous()
        gs, rec["generic_same_shape"] = run(ctx, Xs, a.k, 2, _native.PATH_GENERIC, init)
        ws, _ = run(ctx, Xs, a.k, 2, _native.PATH_AUTO, init)
        rec["agreement"] = {"rows": a.n_generic, "max_abs_mean_diff": float(np.abs(ws["means"] - gs["means"]).max()),
                            "max_abs_weight_diff": float(np.abs(ws["weights"] - gs["weights"]).max()),
                            "ll_rel_diff": abs(ws["log_likelihood"] - gs["log_likelihood"]) / abs(gs["log_likelihood"])}
        rec["torch_fp32_em_step_ms"] = torch_step_ms(X, *init)
        del X, Xs
        X2 = mixture(a.n_generic, 256, a.k, 2)
        _, rec["generic_d256"] = run(ctx, X2, a.k, 2, _native.PATH_AUTO, near_start(X2, a.k))
    rec["card_after"] = card()
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
