"""Child process of tests/test_gpu_ranks_silhouette_multi.py: b2k_silhouette_multi and, for each model, b2k_silhouette
at R ranks as threads of this process, all on cuda:0, through the in-process NCCL stand-in, with the harness of
tests/_ranks_child.py.

    python tests/_ranks_child_silhouette_multi.py silhouette_multi <R> <out.pkl>
"""
from __future__ import annotations

import os
import pickle
import sys
import traceback

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import _ranks_child as rc  # noqa: E402
from _ranks_child_silhouette import shard_sizes  # noqa: E402

# (name, d, Ks, metric, kernel_path)
CASES = [("wg_d32", 32, (9, 3, 130), "squaredEuclidean", 2), ("gen_d7", 7, (9, 2, 70), "squaredEuclidean", 1),
         ("wg_cos", 64, (5, 17), "cosine", 2)]


def data(d, Ks, seed, n=3000):
    """Blobs and one labelling per K; in each, one cluster (id 1000 + m) holds the last 40 rows only, so that at R > 1
    it lives on the last rank only."""
    rng = np.random.default_rng(seed)
    mu = rng.normal(size=(8, d)) * 3
    blob = rng.integers(0, 8, n)
    X = (mu[blob] + rng.normal(size=(n, d))).astype(np.float32)
    ids = []
    for m, K in enumerate(Ks):
        lab = ((blob * 7 + np.arange(n) * (m + 1)) % (K - 1)).astype(np.int64) - 1
        lab[-40:] = 1000 + m
        ids.append(lab)
    return X, ids


def _parts(X, ids, R):
    sz = shard_sizes(R, len(X))
    cols = {"X": rc.split(X, sz)}
    for m, i in enumerate(ids):
        cols[f"ids{m}"] = rc.split(i, sz)
    return [{k: v[r] for k, v in cols.items()} for r in range(R)]


def _fn(M, metric, path):
    def f(ctx, a):
        ctx.set_option("kernel_path", path)
        ids = [a[f"ids{m}"] for m in range(M)]
        return {"multi": ctx.silhouette_multi(a["X"], ids, metric),
                "single": [ctx.silhouette(a["X"], i, metric) for i in ids]}
    return f


def _cases(R):
    cases = {}
    for name, d, Ks, metric, path in CASES:
        X, ids = data(d, Ks, seed=d + len(Ks))
        cases[name] = (_parts(X, ids, R), _fn(len(Ks), metric, path))
    X, ids = data(16, (6, 4), seed=3)
    Xb = X.copy()
    Xb[-5, 3] = np.inf   # on the last rank only
    cases["nonfinite"] = (_parts(Xb, ids, R), _fn(2, "squaredEuclidean", 0))
    one = [ids[0], np.zeros_like(ids[1])]
    cases["one_cluster"] = (_parts(X, one, R), _fn(2, "squaredEuclidean", 0))
    return cases


def main(R, out_path):
    res = {}
    for name, (parts, fn) in _cases(R).items():
        try:
            outs, errs, trace, gerr, secs = rc.run_ranks(R, parts, fn)
            res[name] = {"outs": outs, "errs": errs, "group_error": gerr, "secs": secs}
        except Exception:  # noqa: BLE001 - a harness failure is the parent's to report
            res[name] = {"harness_error": traceback.format_exc()}
    with open(out_path, "wb") as f:
        pickle.dump(res, f)


if __name__ == "__main__":
    sys.path.insert(0, rc.ROOT)
    main(int(sys.argv[2]), sys.argv[3])
