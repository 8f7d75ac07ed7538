"""Sparse logistic regression on one GPU: seeded data generated on the device, the CSR passes timed with CUDA events
(option time_kernels), the bytes each pass must move counted from the data, and two baselines: one fp32 and one fp64
torch.sparse_csr_tensor autograd evaluation on the same rows, and held-out accuracy against scikit-learn on a
subsample.  Prints the card's name and power limit and one JSON line per workload.

    python bench_logreg_sparse.py [--small]

Workloads: binomial n = 10 M, d = 2^18, 64 entries per row; multinomial K = 20, n = 1 M, d = 2^17, about 100 entries per
row.  Column popularity is skewed (u^3 over the columns, a power law), labels come from a planted sparse model.  The
last 1 % of the rows are held out: the device fit and scikit-learn's are both scored on them and neither trains on them;
the device fit trains on all the other rows, scikit-learn on the first 1 M."""
from __future__ import annotations

import argparse
import json
import subprocess
import time

import numpy as np
import torch

from spark_rapids_ml_b200 import _native

HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet


def gen(n, d, per_row, K, seed):
    """Device CSR (indptr, indices, values), labels, on cuda:0: per row `per_row` distinct sorted columns."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    u = torch.rand((n, per_row), generator=g, device="cuda")
    cols = torch.sort(((d - per_row) * u ** 3).long(), dim=1).values + torch.arange(per_row, device="cuda")
    vals = torch.randn((n, per_row), generator=g, device="cuda")
    del u
    wt = torch.randn((K, d), generator=g, device="cuda", dtype=torch.float64)
    wt *= (torch.rand((K, d), generator=g, device="cuda") < 0.05)
    m = torch.stack([(wt[k][cols] * vals.double()).sum(1) for k in range(K)], 1)
    noise = -torch.log(-torch.log(torch.rand((n, K), generator=g, device="cuda", dtype=torch.float64)))
    y = (m + noise).argmax(1).float() if K > 2 else (m[:, 0] + noise[:, 0] - noise[:, 1] > 0).float()
    indptr = torch.arange(0, n * per_row + 1, per_row, device="cuda", dtype=torch.int64)
    return (indptr, cols.reshape(-1).int(), vals.reshape(-1).contiguous()), y


def counted_bytes(X, n, kp):
    """Bytes the rows pass and the CSC pass must move: streamed indices and values (4 + 4 per entry, 8 per row of
    indptr), R and loss written and read once, W gathered once per distinct column; the CSC pass streams 12 bytes per
    entry and gathers one 32-byte sector per distinct R sector per column."""
    indptr, idx, val = X
    nnz = idx.numel()
    rows_b = 8 * (n + 1) + 8 * nnz + 2 * 8 * n * (kp + 1) + 8 * kp * int(torch.unique(idx).numel())
    row = torch.repeat_interleave(torch.arange(n, device="cuda"), indptr[1:] - indptr[:-1])
    sectors = 0
    for k0 in range(0, kp, max(1, 4 // kp) if kp < 4 else 4):   # 4 doubles per sector
        sec = (row * kp + k0) * 8 // 32
        key = idx.long() * ((n * kp * 8) // 32 + 1) + sec
        sectors += int(torch.unique(key).numel())
        if kp < 4:
            break
    csc_b = 12 * nnz + 32 * sectors
    del row
    return rows_b, csc_b


def timed(fn, reps=3):
    best = float("inf")
    out = None
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        best = min(best, time.perf_counter() - t0)
    return best * 1e3, out


def torch_eval_ms(X, n, d, y, kp, dtype):
    indptr, idx, val = X
    A = torch.sparse_csr_tensor(indptr, idx.long(), val.to(dtype), size=(n, d))
    W = torch.zeros((d, kp), dtype=dtype, device="cuda", requires_grad=True)
    b = torch.zeros(kp, dtype=dtype, device="cuda", requires_grad=True)

    def run():
        W.grad = None
        b.grad = None
        m = A @ W + b
        if kp == 1:
            loss = torch.nn.functional.binary_cross_entropy_with_logits(m[:, 0], y.to(dtype))
        else:
            loss = torch.nn.functional.cross_entropy(m, y.long())
        loss.backward()
        return float(loss)

    run()
    return timed(run)[0]


def split(X, y, m):
    """Rows [0, m) of a device CSR and its labels (views)."""
    indptr, idx, val = X
    e = int(indptr[m])
    return (indptr[: m + 1], idx[:e], val[:e]), y[:m].contiguous()


def accuracy(X, y, rows, d, coef, icpt, classes):
    import scipy.sparse as sp

    indptr, idx, val = [t.cpu().numpy() for t in X]
    A = sp.csr_matrix((val, idx, indptr - indptr[0]), shape=(len(indptr) - 1, d))[rows]
    M = A @ coef.T + icpt
    pred = classes[(M[:, 0] > 0).astype(int)] if coef.shape[0] == 1 else classes[M.argmax(1)]
    return float((pred == y.cpu().numpy()[rows]).mean())


def sklearn_accuracy(X, y, d, sk_rows, test, reg):
    """scikit-learn's LogisticRegression (lbfgs, 100 iterations) on the first sk_rows rows, scored on the test rows."""
    import scipy.sparse as sp
    from sklearn.linear_model import LogisticRegression as SK

    indptr, idx, val = [t.cpu().numpy() for t in X]
    yh = y.cpu().numpy()
    A = sp.csr_matrix((val, idx, indptr), shape=(len(yh), d))
    sk = SK(C=1.0 / (reg * sk_rows), max_iter=100).fit(A[:sk_rows], yh[:sk_rows])
    return float((sk.predict(A[test]) == yh[test]).mean())


def kernel_breakdown(ctx, X, d, y, classes, counts, s):
    """Device time per kernel (torch.profiler, CUDA activities) of one fit of two iterations: the CSC build, the moments
    pass (k_csc_pass<1>, <2>), and the evaluations (k_csr_rows<true>, k_csc_pass<0>, k_csc_carry)."""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        ctx.logreg_fit_csr(X, d, y, classes, counts, [dict(s, max_iter=2)])
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        name = e.key.replace("(anonymous namespace)::", "").replace("void ", "").split("(")[0]
        if "RadixSort" in name:
            name = "cub radix sort: " + name.split("::")[-1].split("<")[0]
        if any(k in name for k in ("k_csc", "k_csr", "radix sort")):
            t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
            o = out.setdefault(name, {"calls": 0, "ms": 0.0})
            o["calls"] += int(e.count)
            o["ms"] = round(o["ms"] + t / 1e3, 3)
    return out


def workload(name, n, d, per_row, K, reg, sk_rows, seed):
    kp = 1 if K == 2 else K
    X, y = gen(n, d, per_row, K, seed)
    n_test = n // 100   # the last rows: never seen by either fit
    test = slice(n - n_test, n)
    Xtr, ytr = split(X, y, n - n_test)
    out = {"workload": name, "n": n, "d": d, "nnz": int(X[1].numel()), "K": K}
    with _native.Context(0) as ctx:
        ctx.set_option("time_kernels", 1)
        classes, counts, _ = ctx.logreg_labels(y)
        cls = classes if kp > 1 else classes[:2]
        W, b = np.zeros((kp, d)), np.zeros(kp)
        ctx.logreg_eval_csr(X, d, y, cls, W, b)   # warm-up
        rows_ms, csc_ms, ar_ms, build_ms = [], [], [], []
        for _ in range(3):
            ctx.logreg_eval_csr(X, d, y, cls, W, b)
            st = ctx.stats()
            rows_ms.append(st["last_fused_ms"])
            csc_ms.append(st["last_reduce_ms"])
            ar_ms.append(st["last_allreduce_ms"])
            build_ms.append(st["last_finalize_ms"])
        ev = min(r + c + a for r, c, a in zip(rows_ms, csc_ms, ar_ms))
        rows_b, csc_b = counted_bytes(X, n, kp)
        s = {"reg": reg, "l1_ratio": 0.0, "tol": 1e-6, "max_iter": 30, "fit_intercept": True, "standardization": True,
             "family": "auto"}
        ctr, cnt_tr, _ = ctx.logreg_labels(ytr)
        evals0 = ctx.stats()["generic_launches"]
        t0 = time.perf_counter()
        coef, icpt, iters = ctx.logreg_fit_csr(Xtr, d, ytr, ctr, cnt_tr, [s])[0]
        fit_ms = (time.perf_counter() - t0) * 1e3
        st = ctx.stats()
        evals = st["generic_launches"] - evals0
        pred_ms, _ = timed(lambda: ctx.logreg_predict_csr(X, d, coef, icpt, ctr[:max(2, kp)]))
        # the fit's time less its device evaluations (at the measured evaluation time), CSC build and moments pass:
        # the host's share (optimiser, W transpose and copies, stream synchronisation per evaluation)
        fit_other = fit_ms - evals * ev - st["last_finalize_ms"] - st["last_probe_ms"]
        out.update(rows_pass_ms=min(rows_ms), csc_pass_ms=min(csc_ms), allreduce_ms=min(ar_ms), eval_ms=ev,
                   csc_build_ms=min(build_ms), fit_rows=n - n_test, fit_csc_build_ms=st["last_finalize_ms"],
                   moments_ms=st["last_probe_ms"], fit_ms=fit_ms, fit_iters=iters, fit_evaluations=evals,
                   fit_ms_outside_passes=fit_other, predict_rows_per_s=n / (pred_ms / 1e3), rows_pass_bytes=rows_b,
                   csc_pass_bytes=csc_b, eval_bytes_per_s=(rows_b + csc_b) / (ev / 1e3),
                   eval_share_of_hbm=(rows_b + csc_b) / (ev / 1e3) / HBM_BYTES_PER_S,
                   heldout_rows=n_test, heldout_acc=accuracy(X, y, test, d, coef, icpt, ctr[:max(2, kp)]))
        ctx.set_option("time_kernels", 0)
        out["kernels_two_iteration_fit"] = kernel_breakdown(ctx, Xtr, d, ytr, ctr, cnt_tr, s)
    out["torch_fp32_eval_ms"] = torch_eval_ms(X, n, d, y, kp, torch.float32)
    out["torch_fp64_eval_ms"] = torch_eval_ms(X, n, d, y, kp, torch.float64)
    if sk_rows:
        out["sklearn_rows"] = sk_rows
        out["sklearn_heldout_acc"] = sklearn_accuracy(X, y, d, sk_rows, test, reg)
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--small", action="store_true", help="tiny sizes: a rehearsal of the script, not a measurement")
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    print(json.dumps({"card": card}))
    if a.small:
        specs = [("binomial", 20000, 1 << 12, 16, 2, 1e-3, 5000, 1), ("multinomial", 5000, 1 << 11, 20, 5, 1e-3, 0, 2)]
    else:
        specs = [("binomial", 10_000_000, 1 << 18, 64, 2, 1e-6, 1_000_000, 1),
                 ("multinomial", 1_000_000, 1 << 17, 100, 20, 1e-5, 0, 2)]
    for spec in specs:
        print(json.dumps(workload(*spec)), flush=True)


if __name__ == "__main__":
    main()
