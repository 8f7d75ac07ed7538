"""Child process of tests/test_gpu_ranks_logreg_sparse.py: the sparse logistic fit at R ranks as threads of this process,
all on cuda:0, through the in-process NCCL stand-in (the rank harness of tests/_ranks_child.py).  Pickles, per case,
each rank's fit bits or error text and the one-rank fit on the concatenated rows.

    python tests/_ranks_child_logreg_sparse.py <R> <out.pkl>
"""
from __future__ import annotations

import os
import pickle
import sys
import traceback

import numpy as np
import scipy.sparse as sp

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import _ranks_child as rc  # noqa: E402
import logreg_sparse_oracle as so  # noqa: E402

SETTING = {"reg": 0.01, "l1_ratio": 0.0, "tol": 1e-10, "max_iter": 200, "fit_intercept": True,
           "standardization": True, "family": "auto"}


def data(n, d, K, seed, empty_rows=()):
    X = so.random_csr(n, d, 6, seed, zipf=1.4).tolil()
    for r in empty_rows:
        X[r, :] = 0.0
    X = sp.csr_matrix(X, dtype=np.float32)
    X.eliminate_zeros()
    rng = np.random.default_rng(seed)
    y = (np.asarray(X @ rng.normal(size=(K, d)).T) + rng.gumbel(size=(n, K))).argmax(1).astype(np.float32)
    return X, y


def shard_sizes(n, R):   # uneven shards; the last rank's rows are all empty in the data
    return [n - 50, 50] if R == 2 else [n - 90, 40, 50]


def _part(X, y, r0, r1):
    S = X[r0:r1]
    return {"indptr": S.indptr.astype(np.int64), "indices": S.indices.astype(np.int32),
            "values": S.data.astype(np.float32), "y": y[r0:r1]}


def _fit_fn(d):
    def fn(ctx, a):
        X = (a["indptr"], a["indices"], a["values"])
        classes, counts, _ = ctx.logreg_labels(a["y"])
        coef, icpt, it = ctx.logreg_fit_csr(X, d, a["y"], classes, counts, [SETTING])[0]
        return {"bits": coef.tobytes() + icpt.tobytes(), "coef": coef, "icpt": icpt, "iters": it}
    return fn


def _cases(R):
    cases = {}
    for name, n, d, K in [("binomial", 3000, 400, 2), ("multinomial", 3000, 200, 4)]:
        sz = shard_sizes(n, R)
        X, y = data(n, d, K, seed=K, empty_rows=range(n - 50, n))
        bounds = np.concatenate([[0], np.cumsum(sz)])
        parts = [_part(X, y, bounds[i], bounds[i + 1]) for i in range(R)]
        cases[name] = (parts, _part(X, y, 0, n), _fit_fn(d))
    X, y = data(300, 20, 2, seed=9)
    empty = [_part(X, y, 0, 300)] + [_part(X, y, 300, 300) for _ in range(R - 1)]
    cases["fail_empty_rank"] = (empty, None, _fit_fn(20))
    return cases


def main(R, out_path):
    sys.path.insert(0, rc.ROOT)
    res = {}
    for name, (parts, one, fn) in _cases(R).items():
        try:
            outs, errs, trace, gerr, secs = rc.run_ranks(R, parts, fn)
            single = rc.run_single(one, fn) if one is not None else None
            res[name] = {"outs": outs, "errs": errs, "group_error": gerr, "secs": secs, "single": single}
        except Exception:  # noqa: BLE001 - a harness failure is the parent's to report
            res[name] = {"harness_error": traceback.format_exc()}
    with open(out_path, "wb") as f:
        pickle.dump(res, f)


if __name__ == "__main__":
    main(int(sys.argv[1]), sys.argv[2])
