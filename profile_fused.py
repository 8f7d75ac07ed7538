"""Per-phase cycle profile of the 3xTF32 fused Lloyd pass at BASELINE cfg2 (k = 64, d = 128, 10 M float32 rows).

Runs one Lloyd step with option profile_fused (a separately compiled instantiation of k_wg_assign that counts clock64()
cycles per warp and phase, csrc/b2k_wg.cuh WG_P_*) on the inputs bench.py uses, and prints cycles per 128-row tile:
the mean over the 8 consumer warps of every CTA, and the producer warp separately.  The card's name and power limit are
read in the same run.  Prints a table, then ONE JSON line.

  python profile_fused.py [--rows 10000000] [--d 128] [--k 64] [--warmup 3]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench_pca import _card  # noqa: E402

CONSUMER = ["X wait", "centre wait", "hand-off wait", "A load + split", "MMA issue + drain", "epilogue", "sort",
            "column sums"]
PRODUCER = ["X slot wait", "centre stage wait", "issue"]
TILE_ROWS = 128


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--d", type=int, default=128)
    ap.add_argument("--k", type=int, default=64)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()

    import numpy as np
    import torch

    from bench import make_blobs_device
    from spark_rapids_ml_b200 import _native

    dev = torch.device("cuda", 0)
    X, _ = make_blobs_device(torch, dev, a.rows, a.d, a.k, 0)
    C0 = X[: a.k].clone()   # bench.py's cfg2 initialisation (first k rows)
    with _native.Context(0) as ctx:
        ctx.set_option("kernel_path", 2)
        ctx.kmeans_lloyd(X, C0.clone(), a.warmup, -1.0)
        ctx.set_option("profile_fused", 1)
        ctx.kmeans_lloyd(X, C0.clone(), 1, -1.0)
        ctx.set_option("profile_fused", 0)
        prof = ctx.fused_profile().astype(np.float64)   # [grid, warps, 8]
    grid = prof.shape[0]
    ntiles = -(-a.rows // TILE_ROWS)
    tiles = np.array([len(range(b, ntiles, grid)) for b in range(grid)], dtype=np.float64)
    per_tile = prof / tiles[:, None, None]
    cons = per_tile[:, :8, :].mean(axis=(0, 1))
    prod = per_tile[:, 8, :3].mean(axis=0)
    rec = {"shape": {"n": a.rows, "d": a.d, "k": a.k}, "grid": grid, "tiles_per_cta": float(tiles.mean()),
           "consumer_cycles_per_tile": {nm: round(float(v)) for nm, v in zip(CONSUMER, cons)},
           "consumer_total": round(float(cons.sum())),
           "producer_cycles_per_tile": {nm: round(float(v)) for nm, v in zip(PRODUCER, prod)},
           "producer_total": round(float(prod.sum())), **_card()}
    print(f"{rec['gpu']}, power limit {rec['power_limit']}; grid {grid}, {rec['tiles_per_cta']:.1f} tiles per CTA")
    print("consumer warps (mean), cycles per tile:")
    for nm, v in rec["consumer_cycles_per_tile"].items():
        print(f"  {nm:20s} {v:8d}")
    print(f"  {'total':20s} {rec['consumer_total']:8d}")
    print("producer warp, cycles per tile:")
    for nm, v in rec["producer_cycles_per_tile"].items():
        print(f"  {nm:20s} {v:8d}")
    print(f"  {'total':20s} {rec['producer_total']:8d}")
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
