"""ALS benchmark: b2k_als_fit on seeded synthetic power-law ratings on one GPU (default 1 M users x 200 k items x 100 M
ratings, both sides' degrees Zipf-like), at rank 10, 64 and 128, explicit and implicit.  Prints one JSON record with,
per setting: the mean device time per half-step of the normal-equation pass, the Cholesky solve pass, the factor
allgather and (implicit) the Y^T Y pass (CUDA events inside the library, option time_kernels); the setup time (check,
id maps, redistribution, sorts); the whole fit time at --max-iter; the normal-equation pass's fp64 rate (r (r + 1) / 2
+ r FMAs per rating, 2 FLOPs each) against the data-sheet fp64 figures of the H100 SXM (34 TFLOP/s FMA, 67 TFLOP/s
tensor) and its gather bytes (one source row of r fp32 plus the 8-byte index and rating per rating) against 3.35 TB/s;
and the card's name and power limit read in the same run.

    python bench_als.py [--users 1000000] [--items 200000] [--ratings 100000000] [--ranks 10,64,128] [--max-iter 5]
"""
import argparse
import json
import subprocess
import time

import torch

from spark_rapids_ml_b200 import _native

HBM = 3.35e12
FP64_FMA = 34e12
FP64_TC = 67e12


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"unavailable: {e}"


def ratings(n_users, n_items, n, seed):
    """Power-law (Pareto 1.2) degrees on both sides, shuffled ids, ratings 1..5 (explicit) or normal (implicit)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    pu = torch.randperm(n_users, device="cuda", generator=g)
    pi = torch.randperm(n_items, device="cuda", generator=g)

    def draw(m):
        x = torch.rand(n, device="cuda", generator=g, dtype=torch.float64)
        k = ((x.clamp_min(1e-12) ** (-1.0 / 1.2) - 1.0) * (m / 50.0)).clamp_max(m - 1).long()
        return k

    u = pu[draw(n_users)].double()
    i = pi[draw(n_items)].double()
    r = torch.randint(1, 6, (n,), device="cuda", generator=g).float()
    rn = torch.randn(n, device="cuda", generator=g).float() * 2
    return u, i, r, rn


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--users", type=int, default=1_000_000)
    ap.add_argument("--items", type=int, default=200_000)
    ap.add_argument("--ratings", type=int, default=100_000_000)
    ap.add_argument("--ranks", default="10,64,128")
    ap.add_argument("--max-iter", type=int, default=5)
    a = ap.parse_args()
    u, i, r, rn = ratings(a.users, a.items, a.ratings, 0)
    rec = {"bench": "als", "card": card(), "users_drawn": a.users, "items_drawn": a.items, "ratings": a.ratings,
           "max_iter": a.max_iter, "runs": []}
    with _native.Context(0) as ctx:
        ctx.set_option("time_kernels", 1)
        ctx.als_fit(u[:100000], i[:100000], r[:100000], rank=10, max_iter=1)   # warm-up: module load, pools
        for rank in [int(x) for x in a.ranks.split(",")]:
            for implicit in (False, True):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                out = ctx.als_fit(u, i, rn if implicit else r, rank=rank, max_iter=a.max_iter, reg_param=0.1,
                                  implicit_prefs=implicit, alpha=1.0, seed=1)
                torch.cuda.synchronize()
                fit_s = time.perf_counter() - t0
                st = ctx.stats()
                U, I = out["user_ids"].shape[0], out["item_ids"].shape[0]
                finite = bool(torch.isfinite(out["user_factors"]).all() and torch.isfinite(out["item_factors"]).all())
                del out
                ne_ms = st["last_fused_ms"]
                flops = 2.0 * a.ratings * (rank * (rank + 1) / 2 + rank)   # per half-step: every rating once
                gbytes = a.ratings * (4.0 * rank + 8.0)
                t_flop, t_byte = flops / FP64_FMA, gbytes / HBM
                rec["runs"].append({
                    "rank": rank, "implicit": implicit, "users": U, "items": I, "factors_finite": finite,
                    "normal_eq_ms_per_half_step": round(ne_ms, 3),
                    "solve_ms_per_half_step": round(st["last_finalize_ms"], 3),
                    "allgather_ms_per_half_step": round(st["last_allreduce_ms"], 3),
                    "gram_ms_per_half_step": round(st["last_reduce_ms"], 3),
                    "setup_ms": round(st["last_probe_ms"], 1),
                    "fit_s": round(fit_s, 3),
                    "normal_eq_fp64_tflops": round(flops / (ne_ms * 1e-3) / 1e12, 2) if ne_ms > 0 else None,
                    "normal_eq_share_of_fp64_fma_peak": round(t_flop / (ne_ms * 1e-3), 3) if ne_ms > 0 else None,
                    "normal_eq_share_of_fp64_tensor_peak": round(flops / FP64_TC / (ne_ms * 1e-3), 3) if ne_ms else None,
                    "normal_eq_gather_tb_s": round(gbytes / (ne_ms * 1e-3) / 1e12, 3) if ne_ms > 0 else None,
                    "normal_eq_larger_bound": "fp64 FMA" if t_flop >= t_byte else "HBM",
                    "normal_eq_share_of_larger_bound": round(max(t_flop, t_byte) / (ne_ms * 1e-3), 3) if ne_ms else None,
                })
                print(json.dumps(rec["runs"][-1]), flush=True)
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
