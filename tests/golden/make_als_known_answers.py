"""Writes als_known_answers.json: ALS fits derived by hand from the rules in include/b2kmeans.h, with plain Python
floats (no numpy, no solver).

- constant_rank1: rank 1, every (user, item) pair of m users x k items rated c, start factors all 1.  The item
  half-step has A = m, b = c m, n = m, so every item is c m / (m + reg m) = c / (1 + reg) (= v); the user half-step has
  A = k v^2, b = c k v, n = k, so every user is c v / (v^2 + reg).  Each later iteration repeats the two steps from the
  new factors.
- implicit_rank1: the same in implicit mode with c > 0: c1 = alpha c, the item half-step has Y^T Y = m u^2,
  A = m u^2 + m c1 u^2, b = m (1 + c1) u, n = m, so v = (1 + c1) u / ((1 + c1) u^2 + reg); the user half-step likewise
  with k and v.

Every step rounds to fp32 as the device stores it.

    python tests/golden/make_als_known_answers.py
"""
import json
import os
import struct


def f32(x):
    return struct.unpack("f", struct.pack("f", x))[0]


def constant_rank1(m, k, c, reg, iters):
    u, v = 1.0, 0.0
    for _ in range(iters):
        v = f32((c * m * u) / (m * u * u + reg * m))
        u = f32((c * k * v) / (k * v * v + reg * k))
    return {"m": m, "k": k, "c": c, "reg": reg, "iters": iters, "implicit": False, "alpha": 1.0, "user": u, "item": v}


def implicit_rank1(m, k, c, reg, alpha, iters):
    c1 = alpha * abs(c)
    u, v = 1.0, 0.0
    for _ in range(iters):
        v = f32((m * (1 + c1) * u) / (m * u * u + m * c1 * u * u + reg * m))
        u = f32((k * (1 + c1) * v) / (k * v * v + k * c1 * v * v + reg * k))
    return {"m": m, "k": k, "c": c, "reg": reg, "iters": iters, "implicit": True, "alpha": alpha, "user": u, "item": v}


def main():
    cases = {
        "constant_rank1": constant_rank1(4, 3, 2.5, 0.1, 1),
        "constant_rank1_iter3": constant_rank1(5, 2, 4.0, 0.5, 3),
        "implicit_rank1": implicit_rank1(3, 4, 2.0, 0.2, 0.5, 2),
    }
    out = os.path.join(os.path.dirname(os.path.abspath(__file__)), "als_known_answers.json")
    with open(out, "w") as f:
        json.dump(cases, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
