"""fp64 / integer NumPy restatement of the random-forest semantics of include/b2kmeans.h ("random forests").

Every step is the header's: the SplitMix64-style hash, the Poisson(1) bootstrap table, the sampled thresholds, the
feature subsets, exact integer statistics, the gains in fp64 with each operation rounded once in the stated order, the
split and leaf rules, breadth-first numbering and the leaf values.  A forest fitted on the device must equal fit() node
for node, bit for bit.  Trees are grown one at a time here (the device grows them level by level, all trees at once);
the result does not depend on that order.
"""
from __future__ import annotations

import math
from typing import Any, Dict, List, Tuple

import numpy as np

MASK = (1 << 64) - 1
GOLD = 0x9E3779B97F4A7C15
BOOT, SAMPLE, FEAT = 1, 2, 3
POISSON_CDF = np.array([1580030168, 3160060337, 3950075421, 4213413783, 4279248373, 4292415291, 4294609777,
                        4294923276, 4294962463, 4294966817, 4294967252, 4294967292], dtype=np.uint64)
POISSON_CAP = 12
IMPURITIES = ("gini", "entropy", "variance")


def _mix(z: np.ndarray) -> np.ndarray:
    z = z ^ (z >> np.uint64(30))
    z = z * np.uint64(0xBF58476D1CE4E5B9)
    z = z ^ (z >> np.uint64(27))
    z = z * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def rf_hash(seed: int, stream: int, tree: int, index: Any) -> np.ndarray:
    """h(seed, stream, tree, index) for an array of indices (uint64 arithmetic, wrapping)."""
    idx = np.asarray(index, dtype=np.uint64)
    with np.errstate(over="ignore"):
        a = _mix(np.array([(seed + stream * GOLD) & MASK], dtype=np.uint64))
        b = _mix(a + np.uint64((tree * GOLD) & MASK))
        return _mix(b + idx * np.uint64(GOLD))


def poisson(u32: np.ndarray) -> np.ndarray:
    """The least k with u < table[k], else the cap."""
    return np.searchsorted(POISSON_CDF, np.asarray(u32, dtype=np.uint64), side="right").astype(np.int64)


def weights(seed: int, tree: int, n: int, bootstrap: bool) -> np.ndarray:
    if not bootstrap:
        return np.ones(n, dtype=np.int64)
    return poisson(rf_hash(seed, BOOT, tree, np.arange(n, dtype=np.uint64)) >> np.uint64(32))


def sample_rows(seed: int, n: int, max_bins: int) -> np.ndarray:
    M = max(float(max_bins) * max_bins, 10000.0)
    if M >= n:
        return np.arange(n)
    thr = int(math.ldexp(M / n, 64))
    return np.nonzero(rf_hash(seed, SAMPLE, 0, np.arange(n, dtype=np.uint64)) < np.uint64(thr))[0]


def _mid(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    t = ((a.astype(np.float64) + b.astype(np.float64)) / 2.0).astype(np.float32)
    return np.where(t == b, a, t)


def thresholds_of(col: np.ndarray, max_bins: int) -> np.ndarray:
    s = np.sort(np.asarray(col, dtype=np.float32) + np.float32(0.0))
    m = s.size
    v = np.unique(s)
    if v.size <= max_bins:
        return _mid(v[:-1], v[1:]).astype(np.float32)
    p = (np.arange(1, max_bins, dtype=np.int64) * m) // max_bins
    t = _mid(s[p - 1], s[p])
    keep = np.ones(t.size, dtype=bool)
    keep[1:] = t[1:] != t[:-1]
    return t[keep].astype(np.float32)


def thresholds(X: np.ndarray, max_bins: int, seed: int) -> List[np.ndarray]:
    rows = sample_rows(seed, X.shape[0], max_bins)
    return [thresholds_of(X[rows, f], max_bins) for f in range(X.shape[1])]


def bin_matrix(X: np.ndarray, thr: List[np.ndarray]) -> np.ndarray:
    return np.stack([np.searchsorted(thr[f], X[:, f], side="left") for f in range(X.shape[1])], axis=1)


def feature_subset(seed: int, tree: int, heap: int, d: int, k: int) -> np.ndarray:
    perm = list(range(d))
    if k < d:
        h = rf_hash(seed, FEAT, tree, heap * d + np.arange(k, dtype=np.uint64))
        for j in range(k):
            r = j + int(h[j] % np.uint64(d - j))
            perm[j], perm[r] = perm[r], perm[j]
    return np.sort(np.array(perm[:k], dtype=np.int64))


def features_per_node(strategy: str, d: int, n_trees: int, classification: bool) -> int:
    """MLlib's featureSubsetStrategy sizes."""
    s = str(strategy).lower()
    if s == "auto":
        s = "all" if n_trees == 1 else ("sqrt" if classification else "onethird")
    if s == "all":
        return d
    if s == "sqrt":
        return int(math.ceil(math.sqrt(d)))
    if s == "log2":
        return max(1, int(math.ceil(math.log2(d))))
    if s == "onethird":
        return int(math.ceil(d / 3.0))
    try:
        iv = int(s)
        if 1 <= iv:
            return min(iv, d)
        raise ValueError(s)
    except ValueError:
        fv = float(s)
        if 0.0 < fv <= 1.0:
            return int(math.ceil(fv * d))
        raise ValueError(f"featureSubsetStrategy given invalid value {strategy}")


def log2(p: np.ndarray) -> np.ndarray:
    """The header's L(p), in + - * / only."""
    m, e = np.frexp(np.asarray(p, dtype=np.float64))
    low = m < 0.7071067811865476
    m = np.where(low, m * 2.0, m)
    e = np.where(low, e - 1, e)
    z = (m - 1.0) / (m + 1.0)
    z2 = z * z
    a = np.full_like(z, 1.0 / 25.0)
    for i in range(11, -1, -1):
        a = a * z2
        a = a + 1.0 / float(2 * i + 1)
    lv = z * a
    lv = lv * 2.0
    lv = lv * 1.4426950408889634
    return lv + e.astype(np.float64)


def impurity(c: np.ndarray, N: np.ndarray, imp: str) -> np.ndarray:
    """c [..., V] int64 counts, N [...] -> fp64 impurity, classes summed in order."""
    Nd = np.asarray(N, dtype=np.float64)
    s = np.zeros(Nd.shape, dtype=np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        for k in range(c.shape[-1]):
            ck = c[..., k]
            p = ck.astype(np.float64) / Nd
            if imp == "gini":
                t = p * p
                s = np.where(ck > 0, s + t, s)
            else:
                t = p * log2(np.where(ck > 0, p, 1.0))
                s = np.where(ck > 0, s - t, s)
    return 1.0 - s if imp == "gini" else s


def _var_gain(SL: np.ndarray, WL: np.ndarray, S: int, W: int, q2: float) -> np.ndarray:
    D = SL.astype(object) * int(W) - int(S) * WL.astype(object)
    g = np.array([float(x) for x in D.ravel()], dtype=np.float64).reshape(SL.shape)
    g = g * g
    with np.errstate(divide="ignore", invalid="ignore"):
        den = WL.astype(np.float64) * (W - WL).astype(np.float64)
        g = g / den
        g = g / float(W)
        g = g / float(W)
    return g * q2


def label_grid(y: np.ndarray) -> Tuple[np.ndarray, float]:
    """(y_q, q): y_q = rint(y 2^(24-e)), 2^(e-1) < max|y| <= 2^e."""
    ym = float(np.max(np.abs(y.astype(np.float32)))) if y.size else 0.0
    if ym == 0.0:
        return np.zeros(y.shape, dtype=np.int64), 1.0
    m, e = math.frexp(ym)
    if m == 0.5:
        e -= 1
    return np.rint(y.astype(np.float64) * math.ldexp(1.0, 24 - e)).astype(np.int64), math.ldexp(1.0, e - 24)


def fit(X: np.ndarray, y: np.ndarray, *, n_trees: int = 20, max_depth: int = 5, max_bins: int = 32,
        min_instances: int = 1, features_per_node: int = 0, bootstrap: bool = True, impurity_name: str = "gini",
        min_info_gain: float = 0.0, seed: int = 0) -> Dict[str, Any]:
    """The forest as b2k_rf_fit / Context.rf_fit return it (the rows in global order)."""
    X = np.ascontiguousarray(X, dtype=np.float32)
    y = np.asarray(y, dtype=np.float32)
    n, d = X.shape
    k = features_per_node or d
    regression = impurity_name == "variance"
    if regression:
        lab, q = label_grid(y)
        V, n_values = 2, 1
    else:
        lab, q = y.astype(np.int64), 1.0
        V = n_values = int(lab.max()) + 1
    q2 = q * q
    thr = thresholds(X, max_bins, seed)
    nthr = np.array([t.size for t in thr])
    B = int(nthr.max()) + 1
    bins = bin_matrix(X, thr)

    def stats_of(rows: np.ndarray, w: np.ndarray) -> np.ndarray:
        if regression:
            return np.array([int(w[rows].sum()), int((w[rows] * lab[rows]).sum())], dtype=np.int64)
        return np.bincount(lab[rows], weights=w[rows], minlength=V).astype(np.int64)

    def count_of(st: np.ndarray) -> int:
        return int(st[0]) if regression else int(st.sum())

    def may_split(nd: Dict[str, Any]) -> bool:
        if nd["depth"] >= max_depth or nd["count"] < 2 * min_instances:
            return False
        return regression or int(np.count_nonzero(nd["stat"])) > 1

    out: Dict[str, List[Any]] = {"feature": [], "threshold": [], "children": [], "gain": [], "count": [], "value": []}
    offsets = [0]
    for t in range(n_trees):
        w = weights(seed, t, n, bootstrap)
        live = np.nonzero(w > 0)[0]
        root = {"depth": 0, "heap": 1, "stat": stats_of(live, w), "feature": -1, "threshold": 0.0, "children": (-1, -1),
                "gain": 0.0}
        root["count"] = count_of(root["stat"])
        nodes = [root]
        level = [(0, live)] if may_split(root) else []
        while level:
            nxt = []
            for ni, rows in level:
                nd = nodes[ni]
                feats = feature_subset(seed, t, nd["heap"], d, k)
                sub = bins[rows][:, feats]                                # [m, k]
                slot = np.broadcast_to(np.arange(k), sub.shape)
                if regression:
                    base = (slot * B + sub) * 2
                    wr = np.broadcast_to(w[rows][:, None], sub.shape)
                    sr = np.broadcast_to((w[rows] * lab[rows])[:, None], sub.shape)
                    H = (np.bincount(base.ravel(), weights=wr.ravel(), minlength=k * B * 2)
                         + np.bincount((base + 1).ravel(), weights=sr.ravel(), minlength=k * B * 2))
                else:
                    idx = (slot * B + sub) * V + lab[rows][:, None]
                    wr = np.broadcast_to(w[rows][:, None], sub.shape)
                    H = np.bincount(idx.ravel(), weights=wr.ravel(), minlength=k * B * V)
                H = np.rint(H).astype(np.int64).reshape(k, B, -1)
                cum = np.cumsum(H, axis=1)                               # left statistics of candidate b
                N = nd["count"]
                if regression:
                    WL, SL = cum[..., 0], cum[..., 1]
                    NL = WL
                    g = _var_gain(SL, WL, int(nd["stat"][1]), N, q2)
                else:
                    NL = cum.sum(axis=2)
                    NR = N - NL
                    imp_p = impurity(nd["stat"][None, :], np.array([N]), impurity_name)[0]
                    il = impurity(cum, NL, impurity_name)
                    ir = impurity(nd["stat"][None, None, :] - cum, NR, impurity_name)
                    with np.errstate(divide="ignore", invalid="ignore"):
                        a = NL.astype(np.float64) / float(N)
                        b = NR.astype(np.float64) / float(N)
                        g = (imp_p - a * il) - b * ir
                valid = (NL >= min_instances) & (N - NL >= min_instances)
                valid &= np.arange(B)[None, :] < nthr[feats][:, None]
                g = np.where(valid, g, -np.inf)
                j = int(np.argmax(g.ravel()))
                best = float(g.ravel()[j])
                if not valid.ravel()[j] or not best > 0.0 or best < min_info_gain:
                    continue
                s, bb = divmod(j, B)
                f = int(feats[s])
                left_stat = cum[s, bb].copy()
                li = len(nodes)
                nd.update(feature=f, threshold=float(thr[f][bb]), children=(li, li + 1), gain=best)
                go_left = bins[rows, f] <= bb
                for side, st, r in ((0, left_stat, rows[go_left]), (1, nd["stat"] - left_stat, rows[~go_left])):
                    ch = {"depth": nd["depth"] + 1, "heap": 2 * nd["heap"] + side, "stat": st, "count": count_of(st),
                          "feature": -1, "threshold": 0.0, "children": (-1, -1), "gain": 0.0}
                    nodes.append(ch)
                    if may_split(ch):
                        nxt.append((li + side, r))
            level = nxt
        for nd in nodes:
            out["feature"].append(nd["feature"])
            out["threshold"].append(nd["threshold"])
            out["children"].append(nd["children"])
            out["gain"].append(nd["gain"])
            out["count"].append(nd["count"])
            c = nd["count"]
            if c == 0:
                out["value"].append(np.zeros(n_values))
            elif regression:
                out["value"].append(np.array([(float(nd["stat"][1]) * q) / float(c)]))
            else:
                out["value"].append(nd["stat"].astype(np.float64) / float(c))
        offsets.append(len(out["feature"]))
    return {"tree_offsets": np.array(offsets, dtype=np.int64), "feature": np.array(out["feature"], dtype=np.int32),
            "threshold": np.array(out["threshold"], dtype=np.float32),
            "children": np.array(out["children"], dtype=np.int32).reshape(-1, 2),
            "gain": np.array(out["gain"], dtype=np.float64), "count": np.array(out["count"], dtype=np.int64),
            "value": np.array(out["value"], dtype=np.float64).reshape(-1, n_values), "n_values": n_values,
            "thresholds": thr}


def leaves(X: np.ndarray, forest: Dict[str, Any]) -> np.ndarray:
    """[n, T] the leaf (forest-wide node index) of each row in each tree, routed by threshold (x <= t goes left)."""
    X = np.asarray(X, dtype=np.float32)
    off = forest["tree_offsets"]
    out = np.zeros((X.shape[0], off.size - 1), dtype=np.int64)
    for t in range(off.size - 1):
        o = int(off[t])
        cur = np.zeros(X.shape[0], dtype=np.int64)
        while True:
            f = forest["feature"][o + cur]
            inner = f >= 0
            if not inner.any():
                break
            xi = X[np.arange(X.shape[0]), np.where(inner, f, 0)]
            left = xi <= forest["threshold"][o + cur]
            ch = forest["children"][o + cur]
            cur = np.where(inner, np.where(left, ch[:, 0], ch[:, 1]), cur)
        out[:, t] = o + cur
    return out


def predict(X: np.ndarray, forest: Dict[str, Any], classification: bool) -> Tuple[Any, Any, np.ndarray]:
    """(raw, prob, pred) as b2k_rf_predict: sums in tree order, fp64."""
    lf = leaves(X, forest)
    val = forest["value"]
    T = lf.shape[1]
    if classification:
        raw = np.zeros((X.shape[0], val.shape[1]), dtype=np.float64)
        for t in range(T):
            raw = raw + val[lf[:, t]]
        tot = np.zeros(X.shape[0], dtype=np.float64)
        for kk in range(raw.shape[1]):
            tot = tot + raw[:, kk]
        with np.errstate(divide="ignore", invalid="ignore"):
            prob = np.where(tot[:, None] != 0.0, raw / tot[:, None], 0.0)
        return raw, prob, np.argmax(raw, axis=1).astype(np.float64)
    acc = np.zeros(X.shape[0], dtype=np.float64)
    for t in range(T):
        acc = acc + val[lf[:, t], 0]
    return None, None, acc / float(T)


def feature_importances(forest: Dict[str, Any], d: int) -> np.ndarray:
    """MLlib's rule: each internal node adds gain * N to its feature; each tree's vector sums to 1; the trees' sum is
    normalised."""
    total = np.zeros(d, dtype=np.float64)
    off = forest["tree_offsets"]
    for t in range(off.size - 1):
        imp = np.zeros(d, dtype=np.float64)
        for i in range(int(off[t]), int(off[t + 1])):
            f = int(forest["feature"][i])
            if f >= 0:
                imp[f] += float(forest["gain"][i]) * float(forest["count"][i])
        s = imp.sum()
        if s > 0:
            total += imp / s
    s = total.sum()
    return total / s if s > 0 else total
