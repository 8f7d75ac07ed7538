"""Child process of tests/test_gpu_ranks_silhouette.py: the silhouette (b2k_silhouette) at R ranks as threads of this
process, all on cuda:0, through the in-process NCCL stand-in, with the harness of tests/_ranks_child.py.

    python tests/_ranks_child_silhouette.py silhouette <R> <out.pkl>
"""
from __future__ import annotations

import os
import pickle
import sys
import traceback

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import _ranks_child as rc  # noqa: E402

# (name, d, K, metric, kernel_path)
SIL_CASES = [("wg_d32", 32, 9, "squaredEuclidean", 2), ("gen_d7", 7, 9, "squaredEuclidean", 1),
             ("wg_cos", 64, 5, "cosine", 2)]


def data(d, K, seed, n=3000):
    """Blobs with ids -1 .. K-2 plus one cluster (id 1000) whose rows all sit at the end, so that at R > 1 it lives on
    the last rank only."""
    rng = np.random.default_rng(seed)
    mu = rng.normal(size=(K, d)) * 3
    lab = rng.integers(0, K - 1, n)
    lab[-40:] = K - 1
    X = (mu[lab] + rng.normal(size=(n, d))).astype(np.float32)
    ids = np.where(lab == K - 1, 1000, lab - 1).astype(np.int64)
    return X, ids


def shard_sizes(R, n):
    """Uneven shards with an empty rank in the middle at R = 3."""
    if R == 2:
        return [n * 6 // 10, n - n * 6 // 10]
    return [n * 7 // 10, 0, n - n * 7 // 10]


def _cases(R):
    cases = {}
    for name, d, K, metric, path in SIL_CASES:
        X, ids = data(d, K, seed=d + K)
        sz = shard_sizes(R, len(X))
        parts = [{"X": a, "ids": i} for a, i in zip(rc.split(X, sz), rc.split(ids, sz))]

        def f(ctx, a, metric=metric, path=path):
            ctx.set_option("kernel_path", path)
            return {"value": ctx.silhouette(a["X"], a["ids"], metric)}

        cases[name] = (parts, {"X": X, "ids": ids}, f)
    X, ids = data(16, 6, seed=3)
    sz = shard_sizes(R, len(X))
    Xb = X.copy()
    Xb[-5, 3] = np.inf   # on the last rank only
    cases["nonfinite"] = ([{"X": a, "ids": i} for a, i in zip(rc.split(Xb, sz), rc.split(ids, sz))], None,
                          lambda ctx, a: {"value": ctx.silhouette(a["X"], a["ids"])})
    one = np.zeros_like(ids)
    cases["one_cluster"] = ([{"X": a, "ids": i} for a, i in zip(rc.split(X, sz), rc.split(one, sz))], None,
                            lambda ctx, a: {"value": ctx.silhouette(a["X"], a["ids"])})
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
