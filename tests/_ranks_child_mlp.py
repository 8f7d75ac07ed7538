"""Child process of tests/test_gpu_ranks_mlp.py: b2k_mlp_eval and b2k_mlp_fit at R ranks as threads of this process,
all on cuda:0, through the in-process NCCL stand-in, with the harness of tests/_ranks_child.py.

    python tests/_ranks_child_mlp.py mlp <R> <out.pkl>
"""
from __future__ import annotations

import os
import pickle
import sys
import traceback

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import _ranks_child as rc  # noqa: E402

# (name, layers, n): the wgmma path (d % 4 == 0) and the generic one
MLP_CASES = [("wg", [16, 9, 3], 2500), ("generic", [3, 5, 4], 1800)]


def data(layers, n, seed):
    rng = np.random.default_rng(seed)
    X = rng.normal(size=(n, layers[0])).astype(np.float32)
    y = rng.integers(0, layers[-1], size=n).astype(np.float32)
    w = rng.normal(size=sum(layers[i] * (layers[i - 1] + 1) for i in range(1, len(layers)))) * 0.5
    return X, y, w


def shard_sizes(R, n):
    # uneven, with a one-row rank
    return [n - n * 4 // 10, n * 4 // 10] if R == 2 else [n - n * 3 // 10 - 1, n * 3 // 10, 1]


def _cases(R):
    cases = {}
    for name, layers, n in MLP_CASES:
        X, y, w = data(layers, n, seed=n)
        parts = [{"X": a, "y": b} for a, b in zip(rc.split(X, shard_sizes(R, n)), rc.split(y, shard_sizes(R, n)))]

        def f(ctx, a, layers=layers, w=w):
            F, g, nt = ctx.mlp_eval(a["X"], a["y"], layers, w)
            fit = ctx.mlp_fit(a["X"], a["y"], layers, max_iter=5, seed=3)
            return {"F": F, "g": g, "nt": nt, "fit": fit}

        cases[name] = (parts, {"X": X, "y": y}, f)
    layers = [4, 3, 2]
    X, y, w = data(layers, 300, seed=1)
    bad_y = y.copy()
    bad_y[-1] = 2.0                      # a label >= C on the last rank only
    bad_X = X.copy()
    bad_X[-1, 0] = np.nan                # a NaN on the last rank only
    for name, Xc, yc in (("bad_label", X, bad_y), ("nan", bad_X, y)):
        p = [{"X": a, "y": b} for a, b in zip(rc.split(Xc, shard_sizes(R, 300)), rc.split(yc, shard_sizes(R, 300)))]
        cases[name] = (p, None, lambda ctx, a, w=w: {"F": ctx.mlp_eval(a["X"], a["y"], [4, 3, 2], w)[0]})
    # kernel_path=2 with X misaligned on the last rank only: the wgmma envelope fails on every rank
    X, y, w = data([8, 3, 2], 300, seed=2)
    p = [{"X": a, "y": b} for a, b in zip(rc.split(X, shard_sizes(R, 300)), rc.split(y, shard_sizes(R, 300)))]

    def misaligned(ctx, a, w=w):
        Xa = a["X"]
        if ctx.rank == ctx.nranks - 1:
            buf = Xa.new_empty(Xa.numel() + 1)
            Xa = buf[1:].view(Xa.shape)
            Xa.copy_(a["X"])
        ctx.set_option("kernel_path", 2)
        return {"F": ctx.mlp_eval(Xa, a["y"], [8, 3, 2], w)[0]}

    cases["misaligned"] = (p, None, misaligned)
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
