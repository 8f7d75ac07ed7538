"""fp64 oracle of bisecting k-means (b2k_bkm_fit / b2k_bkm_predict), restating Spark's BisectingKMeans (euclidean) as
include/b2kmeans.h pins it:

- nodes: the root is 1, the children of i are 2i (left) and 2i + 1 (right); a summary is (n, centre, cost);
- minSize = ceil(m) when m >= 1, else ceil(m n_total);
- per level (level < 63, need = k - 1 at the start): a node is divisible when n >= minSize and cost > EPS n; more than
  `need` divisible nodes keep the `need` largest by n, ties to the lower index; none divisible ends the loop;
- a split of centre c starts at c -/+ 1e-4 ||c|| u, u_j = (splitmix64(splitmix64(seed ^ splitmix64(i)) + j) >> 11)
  2^-53;
- maxIter iterations: every row of a dividing node goes to the nearer existing child (fp64 squared distances from the
  fp32 row, ties left), a child with no rows drops out; summaries about the parent centre p:
  centre = p + S1 / n, cost = max(S2 - ||S1||^2 / n, 0);
- level end: one more reassignment with the final centres; the children with rows (in the last summaries) are the
  next active nodes; need drops by the number of nodes divided;
- leaves in depth-first order, left first; predict descends to the nearer existing child, ties left.
"""
from __future__ import annotations

import math
from typing import Dict, List, Tuple

import numpy as np

EPS = 2.220446049250313e-16
LEVEL_LIMIT = 63
M64 = (1 << 64) - 1


def splitmix64(z: int) -> int:
    z = (z + 0x9E3779B97F4A7C15) & M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


def split_noise(seed: int, i: int, d: int) -> np.ndarray:
    s = splitmix64((seed & M64) ^ splitmix64(i))
    return np.array([(splitmix64((s + j) & M64) >> 11) * 2.0 ** -53 for j in range(d)])


def min_size(min_divisible: float, n_total: int) -> int:
    return int(math.ceil(min_divisible)) if min_divisible >= 1.0 else int(math.ceil(min_divisible * n_total))


def choose(divisible: List[Tuple[int, int]], need: int) -> List[int]:
    """(index, n) of the divisible nodes -> the indices that divide: all of them, or the `need` largest by n (ties to
    the lower index), in index order."""
    if len(divisible) > need:
        divisible = sorted(divisible, key=lambda t: (-t[1], t[0]))[:need]
    return sorted(i for i, _ in divisible)


def summarize(X: np.ndarray, p: np.ndarray) -> Tuple[int, np.ndarray, float]:
    n = X.shape[0]
    if n == 0:
        return 0, p.copy(), 0.0
    D = X - p
    S1 = D.sum(axis=0)
    S2 = float((D * D).sum())
    return n, p + S1 / n, max(S2 - float(S1 @ S1) / n, 0.0)


def sides(X: np.ndarray, cl: np.ndarray, cr: np.ndarray, left_alive: bool = True, right_alive: bool = True
          ) -> Tuple[np.ndarray, np.ndarray]:
    """True = right.  Also the margin dl - dr (signed, fp64)."""
    dl = ((X - cl) ** 2).sum(axis=1)
    dr = ((X - cr) ** 2).sum(axis=1)
    if not right_alive:
        return np.zeros(len(X), bool), dl - dr
    if not left_alive:
        return np.ones(len(X), bool), dl - dr
    return dl > dr, dl - dr


def fit(X: np.ndarray, k: int, max_iter: int = 20, min_divisible: float = 1.0, seed: int = 0) -> Dict:
    """Returns nodes {index: (n, centre, cost)}, leaves (indices in depth-first order), the smallest |dl - dr| /
    (dl + dr) of any side decision (how far the run is from a tie), the levels run and the dividing nodes per level."""
    X = np.asarray(X, dtype=np.float32).astype(np.float64)
    n_total, d = X.shape
    ms = min_size(min_divisible, n_total)
    root = summarize(X, X.mean(axis=0))
    nodes: Dict[int, Tuple[int, np.ndarray, float]] = {1: root}
    assign = np.ones(n_total, dtype=np.int64)
    active = [1]
    need, level = k - 1, 1
    margin = math.inf
    divided_per_level = []
    while active and need > 0 and level < LEVEL_LIMIT:
        div = [(i, nodes[i][0]) for i in active if nodes[i][0] >= ms and nodes[i][2] > EPS * nodes[i][0]]
        if not div:
            break
        dividing = choose(div, need)
        divided_per_level.append(dividing)
        new_active = []
        for i in dividing:
            _, c, _ = nodes[i]
            rows = np.nonzero(assign == i)[0]
            Xi = X[rows]
            u = split_noise(seed, i, d)
            l = 1e-4 * float(np.sqrt(c @ c))
            cen = [c - l * u, c + l * u]
            alive = [True, True]
            summ = None
            for _ in range(max_iter):
                right, m = sides(Xi, cen[0], cen[1], alive[0], alive[1])
                if alive[0] and alive[1] and len(m):
                    tot = ((Xi - cen[0]) ** 2).sum(axis=1) + ((Xi - cen[1]) ** 2).sum(axis=1)
                    rel = np.abs(m) / np.maximum(tot, 1e-300)
                    margin = min(margin, float(rel.min()))
                summ = [summarize(Xi[~right], c), summarize(Xi[right], c)]
                for s in range(2):
                    if summ[s][0] == 0:
                        alive[s] = False
                    else:
                        cen[s] = summ[s][1]
            right, m = sides(Xi, cen[0], cen[1], alive[0], alive[1])
            if alive[0] and alive[1] and len(m):
                tot = ((Xi - cen[0]) ** 2).sum(axis=1) + ((Xi - cen[1]) ** 2).sum(axis=1)
                margin = min(margin, float((np.abs(m) / np.maximum(tot, 1e-300)).min()))
            assign[rows] = np.where(right, 2 * i + 1, 2 * i)
            for s in range(2):
                if summ[s][0] > 0:
                    nodes[2 * i + s] = summ[s]
                    new_active.append(2 * i + s)
        active = sorted(new_active)
        need -= len(dividing)
        level += 1
    return {"nodes": nodes, "leaves": leaves(nodes), "margin": margin, "levels": divided_per_level}


def dfs(nodes) -> List[int]:
    out, stack = [], [1]
    while stack:
        i = stack.pop()
        out.append(i)
        for c in (2 * i + 1, 2 * i):
            if c in nodes:
                stack.append(c)
    return out


def leaves(nodes) -> List[int]:
    return [i for i in dfs(nodes) if 2 * i not in nodes and 2 * i + 1 not in nodes]


def predict(X: np.ndarray, nodes) -> Tuple[np.ndarray, np.ndarray]:
    """Leaf number (depth-first order) and squared distance to that leaf's centre, by descent from the root."""
    X = np.asarray(X, dtype=np.float32).astype(np.float64)
    lv = {i: j for j, i in enumerate(leaves(nodes))}
    lab = np.empty(len(X), dtype=np.int32)
    cost = np.empty(len(X))
    for r, x in enumerate(X):
        i = 1
        while i not in lv:
            a, b = 2 * i, 2 * i + 1
            if a in nodes and b in nodes:
                da = ((x - nodes[a][1]) ** 2).sum()
                db = ((x - nodes[b][1]) ** 2).sum()
                i = a if da <= db else b
            else:
                i = a if a in nodes else b
        lab[r] = lv[i]
        cost[r] = ((x - nodes[i][1]) ** 2).sum()
    return lab, cost


def training_cost(nodes) -> float:
    return float(sum(nodes[i][2] for i in leaves(nodes)))
