"""Writes tests/golden/rf_known_answers.json: known answers of the random-forest semantics of include/b2kmeans.h,
computed here in plain Python integers and decimals, apart from tests/rf_oracle.py's NumPy code:

  hash       h(seed, stream, tree, index) for a few inputs
  poisson    floor(2^32 CDF(k)) of Poisson(1), k = 0..11, from 60-digit decimals, and the weights of a few u values
  subsets    partial Fisher-Yates feature subsets of a few nodes
  thresholds the sampled thresholds of two small columns (midpoint rule and quantile rule)

    python tests/golden/make_rf_known_answers.py
"""
import decimal
import json
import os
import struct

MASK = (1 << 64) - 1
GOLD = 0x9E3779B97F4A7C15


def mix(z):
    z ^= z >> 30
    z = (z * 0xBF58476D1CE4E5B9) & MASK
    z ^= z >> 27
    z = (z * 0x94D049BB133111EB) & MASK
    return z ^ (z >> 31)


def h(seed, stream, tree, index):
    return mix((mix((mix((seed + stream * GOLD) & MASK) + tree * GOLD) & MASK) + index * GOLD) & MASK)


def poisson_table():
    decimal.getcontext().prec = 60
    e = decimal.Decimal(1).exp()
    cdf, term, out = decimal.Decimal(0), decimal.Decimal(1), []
    for k in range(12):
        if k:
            term /= k
        cdf += term / e
        out.append(int((cdf * (1 << 32)).to_integral_value(rounding=decimal.ROUND_FLOOR)))
    return out


def f32(x):
    return struct.unpack("f", struct.pack("f", x))[0]


def mid(a, b):
    t = f32((a + b) / 2.0)
    return a if t == b else t


def thresholds(col, max_bins):
    s = sorted(f32(v) + 0.0 for v in col)
    v = sorted(set(s))
    if len(v) <= max_bins:
        return [mid(v[i], v[i + 1]) for i in range(len(v) - 1)]
    out = []
    for j in range(1, max_bins):
        p = j * len(s) // max_bins
        t = mid(s[p - 1], s[p])
        if not out or out[-1] != t:
            out.append(t)
    return out


def subset(seed, tree, heap, d, k):
    perm = list(range(d))
    for j in range(k if k < d else 0):
        r = j + h(seed, 3, tree, heap * d + j) % (d - j)
        perm[j], perm[r] = perm[r], perm[j]
    return sorted(perm[:k])


def main():
    table = poisson_table()
    us = [0, 1580030167, 1580030168, 3950075420, 4294967291, 4294967292, 4294967295]
    col_a = [3.0, -0.0, 0.0, 1.5, 1.5, 2.25, 7.0, 1e-30, 0.1]
    col_b = [float(i % 37) * 0.37 + (i % 5) * 1e-3 for i in range(200)]
    out = {
        "hash": [{"seed": s, "stream": st, "tree": t, "index": i, "h": h(s, st, t, i)}
                 for s, st, t, i in ((0, 1, 0, 0), (42, 1, 3, 12345), (7, 2, 0, 99), (2**63 + 5, 3, 19, 2**40))],
        "poisson_cdf": table,
        "poisson": [{"u": u, "w": next((k for k, c in enumerate(table) if u < c), 12)} for u in us],
        "subsets": [{"seed": s, "tree": t, "heap": hp, "d": d, "k": k, "features": subset(s, t, hp, d, k)}
                    for s, t, hp, d, k in ((5, 0, 1, 10, 3), (5, 4, 9, 128, 12), (11, 2, 3, 7, 7), (1, 0, 2, 3, 1))],
        "thresholds": [{"col": col_a, "max_bins": 32, "t": thresholds(col_a, 32)},
                       {"col": col_b, "max_bins": 8, "t": thresholds(col_b, 8)}],
    }
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "rf_known_answers.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main()
