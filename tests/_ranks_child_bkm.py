"""Child process of tests/test_gpu_ranks_bkm.py: b2k_bkm_fit at R ranks as threads of this process, all on cuda:0,
through the in-process NCCL stand-in, with the harness of tests/_ranks_child.py.

    python tests/_ranks_child_bkm.py bkm <R> <out.pkl>
"""
from __future__ import annotations

import os
import pickle
import sys
import traceback

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import _ranks_child as rc  # noqa: E402

# (name, d, k, min_divisible)
BKM_CASES = [("d16_k8", 16, 8, 1.0), ("d5_k5_frac", 5, 5, 0.05)]


def data(d, k, seed, n=3000):
    rng = np.random.default_rng(seed)
    means = rng.uniform(-10, 10, size=(k + 2, d))
    z = rng.integers(0, k + 2, size=n)
    return (means[z] + 0.05 * rng.normal(size=(n, d))).astype(np.float32)


def shard_sizes(R, n):
    return [n * 6 // 10, n - n * 6 // 10] if R == 2 else [n * 5 // 10, n * 2 // 10, n - n * 7 // 10]


def _cases(R):
    cases = {}
    for name, d, k, md in BKM_CASES:
        X = data(d, k, seed=d + k)
        parts = [{"X": a} for a in rc.split(X, shard_sizes(R, len(X)))]

        def f(ctx, a, k=k, md=md):
            return {"fit": ctx.bkm_fit(a["X"], k, max_iter=10, min_divisible=md, seed=17)}

        cases[name] = (parts, {"X": X}, f)
    X = data(4, 2, seed=1)
    empty = [{"X": a} for a in rc.split(X, [len(X), 0] if R == 2 else [len(X) - 10, 0, 10])]
    cases["empty"] = (empty, None, lambda ctx, a: {"fit": ctx.bkm_fit(a["X"], 2, max_iter=2)})
    return cases


def main(R, out_path):
    res = {}
    for name, (parts, one, fn) in _cases(R).items():
        try:
            outs, errs, trace, gerr, secs = rc.run_ranks(R, parts, fn)
            single = rc.run_single(one, fn) if one is not None else None
            res[name] = {"outs": outs, "errs": errs, "trace": trace, "group_error": gerr, "secs": secs,
                         "single": single}
        except Exception:  # noqa: BLE001 - a harness failure is the parent's to report
            res[name] = {"harness_error": traceback.format_exc()}
    with open(out_path, "wb") as f:
        pickle.dump(res, f)


if __name__ == "__main__":
    sys.path.insert(0, rc.ROOT)
    main(int(sys.argv[2]), sys.argv[3])
