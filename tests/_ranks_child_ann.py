"""Child process of tests/test_gpu_ranks_ann.py: IVF-Flat (b2k_ivf_search) at R ranks as threads of this process, all
on cuda:0, through the in-process NCCL stand-in, with the harness of tests/_ranks_child.py.

    python tests/_ranks_child_ann.py ann <R> <out.pkl>
"""
from __future__ import annotations

import os
import pickle
import sys
import traceback

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import _ranks_child as rc  # noqa: E402

ANN_INT = [("w16", 16, 10, 2), ("g7", 7, 10, 1)]   # (name, d, k, kernel_path)
NLIST, NPROBE = 12, 3


def query_only_sizes(R, n, nq):
    """Every item on rank 0 and every query on the last rank: the ranks in between hold nothing."""
    return [n] + [0] * (R - 1), [0] * (R - 1) + [nq]


def blobs_data():
    rng = np.random.default_rng(31)
    mu = rng.normal(size=(12, 32)) * 4
    X = (mu[rng.integers(0, 12, 4000)] + rng.normal(size=(4000, 32))).astype(np.float32)
    Q = (mu[rng.integers(0, 12, 150)] + rng.normal(size=(150, 32))).astype(np.float32)
    return X, Q


def _search(ctx, a, k, nlist, nprobe, centers=None, **kw):
    dist, idx, C, lists, probes = ctx.ivf_search(a["X"], a["Q"], k, nlist, nprobe, a.get("ids"), centers=centers,
                                                 return_lists=True, **kw)
    return {"dist": rc._np(dist), "idx": rc._np(idx), "centers": rc._np(C), "lists": rc._np(lists),
            "probes": rc._np(probes)}


def _cases(R):
    cases = {}
    for name, d, k, path in ANN_INT:
        Xi, Qi = rc.knn_int_data(d, seed=d + k)
        X, Q = Xi.astype(np.float32), Qi.astype(np.float32)
        ids = (7 * np.arange(len(X)) + 5).astype(np.int64)
        isz, qsz = rc.knn_sizes(R, len(X), len(Q))
        parts = [{"X": a, "Q": q, "ids": i, "C": X[:NLIST]}
                 for a, q, i in zip(rc.split(X, isz), rc.split(Q, qsz), rc.split(ids, isz))]
        one = {"X": X, "Q": Q, "ids": ids, "C": X[:NLIST]}

        def f(ctx, a, k=k, path=path):
            ctx.set_option("kernel_path", path)
            return _search(ctx, a, k, NLIST, NPROBE, centers=a["C"])

        cases[f"int_{name}"] = (parts, one, f)
    X, Q = blobs_data()
    for name, (isz, qsz) in (("uneven", rc.knn_sizes(R, len(X), len(Q))),
                             ("query_only", query_only_sizes(R, len(X), len(Q)))):
        parts = [{"X": a, "Q": q} for a, q in zip(rc.split(X, isz), rc.split(Q, qsz))]

        def t(ctx, a):
            return _search(ctx, a, 8, 16, 4, n_iters=8)

        cases[f"trained_{name}"] = (parts, {"X": X, "Q": Q}, t)
    # errors, decided on gathered values: a non-finite item on the last rank with items; nlist above the training rows
    isz, qsz = rc.knn_sizes(R, len(X), len(Q))
    Xb = X.copy()
    Xb[len(X) - 3, 5] = np.nan
    cases["nonfinite_item"] = ([{"X": a, "Q": q} for a, q in zip(rc.split(Xb, isz), rc.split(Q, qsz))], None,
                               lambda ctx, a: _search(ctx, a, 8, 16, 4))
    cases["nlist_too_large"] = ([{"X": a, "Q": q} for a, q in zip(rc.split(X, isz), rc.split(Q, qsz))], None,
                                lambda ctx, a: _search(ctx, a, 8, 2001, 4))
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
