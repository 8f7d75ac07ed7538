"""Child process of tests/test_gpu_ranks_rf.py: random forests at R ranks as threads of this process, all on cuda:0,
through the in-process NCCL stand-in, with the rank harness of tests/_ranks_child.py.  Pickles, per case, each rank's
forest (as the model's JSON text) or error text, the collectives the stand-in saw per rank, and the one-rank result on
the concatenated rows.

    python tests/_ranks_child_rf.py <R> <out.pkl>
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


def cls_data(n, d, C, seed):
    rng = np.random.default_rng(seed)
    X = rng.normal(size=(n, d)).astype(np.float32)
    s = X[:, 0] + X[:, 1 % d] + 0.5 * rng.normal(size=n)
    y = np.clip(np.floor((s + 3) / 6 * C), 0, C - 1).astype(np.float32)
    y[0] = C - 1
    return X, y


def reg_data(n, d, seed):
    rng = np.random.default_rng(seed)
    X = rng.normal(size=(n, d)).astype(np.float32)
    return X, (X[:, 0] * 50 - X[:, 2 % d] ** 2 + rng.normal(size=n)).astype(np.float32)


def few_rows_sizes(n, R):   # a rank of a few rows
    return [n - 3, 3] if R == 2 else [n - 7, 4, 3]


# (name, X, y, fit kwargs, kernel_path, shard sizes(n, R))
def case_specs():
    Xc, yc = cls_data(4000, 12, 3, seed=1)
    Xr, yr = reg_data(3000, 8, seed=2)
    Xs, ys = cls_data(30000, 20, 2, seed=3)   # the sample is a strict subset of the rows
    base = dict(n_trees=8, max_depth=6, max_bins=32, features_per_node=4, seed=5)
    return [
        ("gini_cluster", Xc, yc, dict(base, impurity="gini"), 2, rc.sizes),
        ("entropy_generic", Xc, yc, dict(base, impurity="entropy"), 1, rc.sizes),
        ("variance", Xr, yr, dict(base, impurity="variance"), 0, rc.sizes),
        ("sampled_thresholds", Xs, ys, dict(base, max_bins=128, n_trees=3), 0, rc.sizes),
        ("few_rows", Xc, yc, dict(base, impurity="gini", bootstrap=False), 0, few_rows_sizes),
    ]


def _forest_json(out):
    """The forest as the bytes a model would save: every array's raw bits."""
    return b"".join(np.ascontiguousarray(out[k]).tobytes() for k in
                    ("tree_offsets", "feature", "threshold", "children", "gain", "count", "value"))


def _fit_fn(kw, path):
    def fn(ctx, a):
        ctx.set_option("kernel_path", path)
        out = ctx.rf_fit(a["X"], a["y"], **kw)
        return {"bits": _forest_json(out), "path": ctx.stats()["last_path"]}
    return fn


def _cases(R):
    cases = {}
    for name, X, y, kw, path, sz in case_specs():
        s = sz(len(X), R)
        parts = [{"X": a, "y": b} for a, b in zip(rc.split(X, s), rc.split(y, s))]
        cases[name] = (parts, {"X": X, "y": y}, _fit_fn(kw, path))
    X, y = cls_data(600, 5, 2, seed=6)
    s = rc.sizes(len(X), R)
    bad = R - 1

    def parts_with(Xv=None, yv=None):
        p = [{"X": a.copy(), "y": b.copy()} for a, b in zip(rc.split(X, s), rc.split(y, s))]
        if Xv is not None:
            p[bad]["X"][1, 2] = Xv
        if yv is not None:
            p[bad]["y"][2] = yv
        return p

    fit = _fit_fn(dict(n_trees=2, max_depth=3), 0)
    cases["fail_nan"] = (parts_with(Xv=np.nan), None, fit)
    cases["fail_label"] = (parts_with(yv=0.5), None, fit)
    empty = [{"X": a, "y": b} for a, b in zip(rc.split(X, [len(X)] + [0] * (R - 1)), rc.split(y, [len(X)] + [0] * (R - 1)))]
    cases["fail_empty_rank"] = (empty, None, fit)
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
