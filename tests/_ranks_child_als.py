"""Child process of tests/test_gpu_ranks_als.py: b2k_als_fit at R ranks as threads of this process, all on cuda:0,
through the in-process NCCL stand-in, with the harness of tests/_ranks_child.py.

    python tests/_ranks_child_als.py als <R> <out.pkl>
"""
from __future__ import annotations

import os
import pickle
import sys
import traceback

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import _ranks_child as rc  # noqa: E402

# (name, rank, implicit)
ALS_CASES = [("explicit", 10, False), ("implicit", 16, True)]
N = 12000


def data(seed, implicit):
    rng = np.random.default_rng(seed)
    u = np.minimum((rng.pareto(1.2, N) * 30).astype(np.int64), 599) * 5 - 77
    i = np.minimum((rng.pareto(1.2, N) * 20).astype(np.int64), 399) * 3
    r = rng.normal(size=N) * 2 if implicit else rng.integers(1, 6, N).astype(np.float64)
    return u.astype(np.float64), i.astype(np.float64), r.astype(np.float32)


def shard_sizes(R):
    # uneven, with a rank holding no ratings; a user's ratings land on several ranks
    return [N * 6 // 10, N - N * 6 // 10] if R == 2 else [N // 2, 0, N - N // 2]


def _parts(R, u, i, r):
    sz = shard_sizes(R)
    return [{"u": a, "i": b, "r": c} for a, b, c in zip(rc.split(u, sz), rc.split(i, sz), rc.split(r, sz))]


def _cases(R):
    cases = {}
    for name, rank, implicit in ALS_CASES:
        u, i, r = data(rank, implicit)

        def f(ctx, a, rank=rank, implicit=implicit):
            out = ctx.als_fit(a["u"], a["i"], a["r"], rank=rank, max_iter=3, reg_param=0.05, implicit_prefs=implicit,
                              alpha=1.5, seed=9)
            return {k: v.cpu().numpy() for k, v in out.items()}

        cases[name] = (_parts(R, u, i, r), {"u": u, "i": i, "r": r}, f)
    u, i, r = data(1, False)
    bad_u = u.copy()
    bad_u[-1] = 2.0 ** 31       # outside int32, on the last rank only
    bad_r = r.copy()
    bad_r[-1] = np.nan          # a NaN rating on the last rank only
    for name, uu, rr in (("bad_id", bad_u, r), ("nan", u, bad_r)):
        cases[name] = (_parts(R, uu, i, rr), None,
                       lambda ctx, a: {"n": ctx.als_fit(a["u"], a["i"], a["r"], rank=4, max_iter=1)["user_ids"].shape})
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
