"""Child process of tests/test_gpu_ranks_dbscan.py: DBSCAN at R ranks as threads of this process, all on cuda:0, through
the in-process NCCL stand-in, with the rank harness of tests/_ranks_child.py.  Pickles, per case, each rank's outputs
or error text, the collectives the stand-in saw per rank, and the one-rank result on the concatenated rows.

    python tests/_ranks_child_dbscan.py <R> <out.pkl>
"""
from __future__ import annotations

import os
import pickle
import sys
import traceback

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import _ranks_child as rc  # noqa: E402


def blobs(n, d, k, seed, spread=3.0, std=1.0):
    rng = np.random.default_rng(seed)
    C = rng.uniform(-spread, spread, size=(k, d))
    return (C[rng.integers(0, k, size=n)] + std * rng.normal(size=(n, d))).astype(np.float32)


def chain(n):
    X = np.zeros((n, 4), dtype=np.float32)
    X[:, 0] = 9.0 * np.arange(n)
    return X


def empty_rank_sizes(n, R):   # a rank with no rows (and, at R = 3, one smaller than a tile)
    return [n, 0] if R == 2 else [n - 5, 0, 5]


# (name, X, eps, min_samples, metric, kernel_path, shard sizes(n, R))
def case_specs():
    return [
        ("blobs_wgmma", blobs(3000, 16, 6, seed=1), 0.85 * np.sqrt(32), 5, "euclidean", 2, rc.sizes),
        ("blobs_generic", blobs(2000, 6, 5, seed=2), 0.85 * np.sqrt(12), 5, "euclidean", 1, rc.sizes),
        ("blobs_d128", blobs(1500, 128, 6, seed=3), 0.85 * 16.0, 4, "euclidean", 2, rc.sizes),
        ("cosine", blobs(1500, 16, 5, seed=4, spread=1.0, std=0.3) + 2.0, 0.02, 5, "cosine", 0, rc.sizes),
        ("chain", chain(6000), 10.0, 3, "euclidean", 2, rc.sizes),
        ("empty_rank", blobs(1200, 8, 4, seed=5), 0.85 * 4.0, 4, "euclidean", 0, empty_rank_sizes),
        ("empty_rank_generic", blobs(1200, 8, 4, seed=5), 0.85 * 4.0, 4, "euclidean", 1, empty_rank_sizes),
    ]


def _fit_fn(eps, ms, metric, path):
    def fn(ctx, a):
        ctx.set_option("kernel_path", path)
        lab, core, ncl = ctx.dbscan_fit(a["X"], eps, ms, metric)
        return {"labels": lab.cpu().numpy(), "core": core.cpu().numpy(), "n_clusters": ncl,
                "path": ctx.stats()["last_path"]}
    return fn


def _cases(R):
    cases = {}
    for name, X, eps, ms, metric, path, sz in case_specs():
        parts = [{"X": p} for p in rc.split(X, sz(len(X), R))]
        cases[name] = (parts, {"X": X}, _fit_fn(float(eps), ms, metric, path))
    X = blobs(600, 8, 3, seed=6)
    bad = R - 1

    def with_row(row, value):
        p = [{"X": a.copy()} for a in rc.split(X, rc.sizes(len(X), R))]
        p[bad]["X"][row] = value
        return p

    fit = _fit_fn(2.0, 3, "euclidean", 0)
    cases["fail_nan"] = (with_row(2, np.nan), None, fit)
    cases["fail_zero_row_cosine"] = (with_row(1, 0.0), None, _fit_fn(0.1, 3, "cosine", 0))
    cases["fail_bad_eps"] = ([{"X": a} for a in rc.split(X, rc.sizes(len(X), R))], None, _fit_fn(-1.0, 3, "euclidean", 0))
    cases["fail_bad_min_samples"] = ([{"X": a} for a in rc.split(X, rc.sizes(len(X), R))], None,
                                     _fit_fn(1.0, 0, "euclidean", 0))
    pd = [{"X": a} for a in rc.split(X, rc.sizes(len(X), R))]
    pd[bad] = {"X": pd[bad]["X"][:, :7].copy()}
    cases["fail_d_differs"] = (pd, None, fit)
    return cases


def main(R, out_path):
    sys.path.insert(0, rc.ROOT)
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
    main(int(sys.argv[1]), sys.argv[2])
