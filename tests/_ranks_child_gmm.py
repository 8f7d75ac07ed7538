"""Child process of tests/test_gpu_ranks_gmm.py: b2k_gmm_fit at R ranks as threads of this process, all on cuda:0,
through the in-process NCCL stand-in, with the harness of tests/_ranks_child.py.

    python tests/_ranks_child_gmm.py gmm <R> <out.pkl>
"""
from __future__ import annotations

import os
import pickle
import sys
import traceback

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import _ranks_child as rc  # noqa: E402

# (name, d, k, kernel_path)
GMM_CASES = [("wg_d16", 16, 4, 0), ("gen_d5", 5, 3, 1)]


def data(d, k, seed, n=3000):
    rng = np.random.default_rng(seed)
    means = rng.normal(scale=5.0, size=(k, d))
    z = rng.integers(0, k, size=n)
    return (means[z] + rng.normal(size=(n, d))).astype(np.float32)


def dead_component(n=3 * 4096 + 5, seed=4):
    """Tight rows (sigma = 0.05, d = 132) of two live components and an injected third one 50 units from every row, whose
    responsibilities lie far below FLT_MIN: (X, (weights, means, covariances))."""
    d, s = 132, 0.05
    rng = np.random.default_rng(seed)
    e = np.eye(d)
    live = np.stack([e[0], -e[0]])
    X = (live[np.arange(n) % 2] + s * rng.normal(size=(n, d))).astype(np.float32)
    init = (np.array([0.45, 0.45, 0.1]), np.stack([e[0], -e[0], 50.0 * e[1]]), np.stack([np.eye(d) * s * s] * 3))
    return X, init


def shard_sizes(R, n):
    return [n * 6 // 10, n - n * 6 // 10] if R == 2 else [n * 5 // 10, n * 2 // 10, n - n * 7 // 10]


def _cases(R):
    cases = {}
    for name, d, k, path in GMM_CASES:
        X = data(d, k, seed=d + k)
        parts = [{"X": a} for a in rc.split(X, shard_sizes(R, len(X)))]

        def f(ctx, a, k=k, path=path):
            ctx.set_option("kernel_path", path)
            start = ctx.gmm_fit(a["X"], k, max_iter=0, seed=17)
            out = ctx.gmm_fit(a["X"], k, max_iter=6, tol=0.0, seed=17)
            return {"start": start, "fit": out}

        cases[name] = (parts, {"X": X}, f)
    if R == 2:
        # one M step, so both of its allreduces run on every rank of an uneven split.  (A second one is not defined:
        # the step gathers the support-less component onto a few rows, and its density then overflows an fp64.)
        X, init = dead_component()
        parts = [{"X": a} for a in rc.split(X, shard_sizes(R, len(X)))]
        cases["dead"] = (parts, {"X": X},
                         lambda ctx, a: {"fit": ctx.gmm_fit(a["X"], 3, init=init, max_iter=1, tol=0.0)})
    X = data(4, 2, seed=1)
    empty = [{"X": a} for a in rc.split(X, [len(X), 0] if R == 2 else [len(X) - 10, 0, 10])]
    cases["empty"] = (empty, None, lambda ctx, a: {"fit": ctx.gmm_fit(a["X"], 2, max_iter=2)})
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
