"""Writes mlp_known_answers.json: multilayer perceptron evaluations derived by hand from the rules in
include/b2kmeans.h, with plain Python floats (no numpy, no solver).

- zero_weights: every weight 0.  The hidden activations are sigmoid(0) = 1/2, z = 0, p = 1/C, so F = log C, delta_L =
  1/C - onehot(y), and the hidden deltas are 0 (W = 0), so only the last layer has a gradient: dW_L(o, i) = mean of
  delta_L,o * 1/2 and db_L(o) = mean of delta_L,o.
- one_layer: layers [2, 2] (softmax regression), one row each, worked out term by term.

    python tests/golden/make_mlp_known_answers.py
"""
import json
import math
import os


def zero_weights():
    layers = [2, 3, 2]
    X = [[1.0, -2.0], [0.5, 4.0], [3.0, 0.0]]
    y = [0, 1, 1]
    n, C, H = len(X), 2, 3
    P = H * (2 + 1) + C * (H + 1)
    w = [0.0] * P
    F = math.log(C)
    grad = [0.0] * P
    off = H * 3
    for o in range(C):
        m = sum((1.0 / C - (1.0 if y[r] == o else 0.0)) for r in range(n)) / n
        for i in range(H):
            grad[off + i * C + o] = m * 0.5
        grad[off + H * C + o] = m
    return {"name": "zero_weights", "layers": layers, "X": X, "y": y, "w": w, "F": F, "grad": grad}


def one_layer():
    layers = [2, 2]
    X = [[1.0, 2.0]]
    y = [1]
    # W (o, i) at i * 2 + o: W = [[0.5, -1.0], [0.25, 0.0]] (rows o), b = [0.1, -0.2]
    W = [[0.5, -1.0], [0.25, 0.0]]
    b = [0.1, -0.2]
    w = [W[0][0], W[1][0], W[0][1], W[1][1], b[0], b[1]]
    z = [W[o][0] * 1.0 + W[o][1] * 2.0 + b[o] for o in range(2)]   # [-1.4, 0.05]
    m = max(z)
    s = sum(math.exp(v - m) for v in z)
    F = math.log(s) - (z[1] - m)
    p = [math.exp(v - m) / s for v in z]
    d = [p[0] - 0.0, p[1] - 1.0]
    grad = [d[0] * 1.0, d[1] * 1.0, d[0] * 2.0, d[1] * 2.0, d[0], d[1]]
    return {"name": "one_layer", "layers": layers, "X": X, "y": y, "w": w, "F": F, "grad": grad}


if __name__ == "__main__":
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "mlp_known_answers.json"), "w") as f:
        json.dump([zero_weights(), one_layer()], f, indent=1)
