"""fp64 oracle of the multilayer perceptron semantics pinned in include/b2kmeans.h (b2k_mlp_*), restated here.

Weights use Spark's flat layout: for each layer l, W_l (numOut x numIn, column-major: element (o, i) at i numOut + o),
then the numOut biases.  Hidden layers apply the sigmoid; the last layer's output z goes to the softmax with
cross-entropy loss.  F(w) = (1/n) sum -log softmax(z)_y, no regularisation.
"""
import math

import numpy as np

U = 2.0 ** -24   # fp32 unit roundoff


def n_weights(layers):
    return sum(layers[i] * (layers[i - 1] + 1) for i in range(1, len(layers)))


def unpack(layers, w):
    """Flat weights -> [(W_l [numOut, numIn], b_l [numOut])]."""
    w = np.asarray(w, dtype=np.float64)
    out, off = [], 0
    for i in range(1, len(layers)):
        ni, no = layers[i - 1], layers[i]
        W = w[off: off + ni * no].reshape(ni, no).T   # column-major numOut x numIn
        off += ni * no
        b = w[off: off + no]
        off += no
        out.append((W.copy(), b.copy()))
    assert off == w.size
    return out


def pack(params):
    return np.concatenate([np.concatenate([W.T.reshape(-1), b]) for W, b in params])


def sigmoid(z):
    return 1.0 / (1.0 + np.exp(-z))


def forward(layers, w, X):
    """Activations [a_0 = X, a_1, ..., a_{L-1}] and z_L."""
    params = unpack(layers, w)
    a = [np.asarray(X, dtype=np.float64)]
    for W, b in params[:-1]:
        a.append(sigmoid(a[-1] @ W.T + b))
    W, b = params[-1]
    return a, a[-1] @ W.T + b


def softmax(z):
    m = z.max(axis=1, keepdims=True)
    e = np.exp(z - m)
    return e / e.sum(axis=1, keepdims=True)


def eval_fg(layers, w, X, y):
    """F(w) and its gradient in the flat layout."""
    params = unpack(layers, w)
    a, z = forward(layers, w, X)
    n = z.shape[0]
    yi = np.asarray(y).astype(np.int64)
    m = z.max(axis=1, keepdims=True)
    lse = np.log(np.exp(z - m).sum(axis=1)) + m[:, 0]
    F = float(np.mean(lse - z[np.arange(n), yi]))
    delta = softmax(z)
    delta[np.arange(n), yi] -= 1.0
    grads = [None] * len(params)
    for l in range(len(params) - 1, -1, -1):
        grads[l] = (delta.T @ a[l] / n, delta.sum(axis=0) / n)
        if l > 0:
            delta = (delta @ params[l][0]) * a[l] * (1.0 - a[l])
    return F, pack(grads)


RHO = 2.0 ** -24   # fp32 unit roundoff, the scale of every error term below
C_TERM = 12.0      # per product term: the dropped lo.lo and the tf32 rounding of lo
C_TRUNC = 24.0     # per 32-wide chunk: 12 truncated tensor-core accumulations of at most one ulp (2 rho) each
CONF = 6.0         # the bound is CONF times the root-sum-square scale below
TINY = 2.0 ** -126 # a stored fp32 value or a tensor-core operand below this may be flushed to zero


def _chunk_trunc(A, B):
    """sqrt(sum over 32-wide K chunks of (sum_k |A_mk B_nk|)^2) for A [M, K] and B [N, K]."""
    out = np.zeros((A.shape[0], B.shape[0]))
    for c in range(0, A.shape[1], 32):
        out += (np.abs(A[:, c:c + 32]) @ np.abs(B[:, c:c + 32]).T) ** 2
    return np.sqrt(out)


def _product_err(A, B, unit=None):
    """Error scales of the wgmma product A [M, K] . B [N, K]^T -> (variance of the random part, systematic part).
    Random: C_TERM rho per term and rho times the running absolute sum per fp32 addition of a chunk sum (16 per 512-row
    Gram unit, K / 32 in a row product), root-sum-square.  Systematic: the tensor core truncates toward zero, so its 12
    accumulations per chunk shrink every chunk's partial by up to C_TRUNC rho of the chunk's absolute sum; the chunks'
    partials have either sign (root-sum-square over chunks), but the shrink of one output is coherent across rows."""
    K = A.shape[1]
    v = (C_TERM * RHO) ** 2 * ((A ** 2) @ (B ** 2).T)
    span = unit or K
    for c in range(0, K, span):
        s1 = np.abs(A[:, c:c + span]) @ np.abs(B[:, c:c + span]).T
        v += RHO ** 2 * (min(span, K - c) / 32.0) * s1 ** 2
    return v, C_TRUNC * RHO * _chunk_trunc(A, B)


def _forward_err(params, a, z):
    """(variance, systematic) error scales of the stored activations [a_0 .. a_{L-1}] and of the stored z."""
    va, sa = [np.zeros_like(a[0])], [np.zeros_like(a[0])]
    for l, (W, b) in enumerate(params[:-1]):
        vp, sp = _product_err(a[l], W)
        vz, sz = vp + va[l] @ (W ** 2).T, sp + sa[l] @ np.abs(W).T
        s = a[l + 1] * (1.0 - a[l + 1])
        va.append(s ** 2 * vz + (RHO * a[l + 1]) ** 2 + TINY ** 2)
        sa.append(s * sz)
    W, b = params[-1]
    vp, sp = _product_err(a[-1], W)
    vz = vp + va[-1] @ (W ** 2).T + (RHO * z) ** 2 + TINY ** 2   # z stored in fp32
    sz = sp + sa[-1] @ np.abs(W).T
    return va, sa, vz, sz


def z_bound(layers, w, X):
    """z and the bound on |z_device - z| per row and class for the wgmma path (the forward half of eval_bound, with the
    exact shift of the fp32 weights)."""
    params = unpack(layers, w)
    a, z = forward(layers, w, X)
    z32 = forward(layers, weights_fp32(layers, w), X)[1]
    _, _, vz, sz = _forward_err(params, a, z)
    return z, CONF * np.sqrt(vz) + sz + np.abs(z32 - z)


def eval_bound(layers, w, X, y):
    """Bound on |F_device - F| and per weight on |grad_device - grad| for the wgmma path (3xTF32 products, fp32
    activations and deltas, fp32 weights, fp32 sums of 32-row chunks per 512-row Gram unit).

    Each error is carried as two scales.  Random (independent rounding of either sign, root-sum-square): C_TERM rho
    per product term (the dropped lo.lo and the tf32 rounding of lo), rho times the running absolute sum per fp32
    addition of a chunk sum, and rho of every stored fp32 value plus an absolute 2^-126, since values that small may be
    flushed to zero (saturated sigmoids give deltas there).  Systematic (the tensor core's truncation toward zero,
    C_TRUNC rho of each chunk's absolute sum, coherent across rows).  Both pass through the weights, the sigmoid's slope
    a (1 - a) and the softmax (dp_c = p_c (dz_c - sum_j p_j dz_j)); the random scales add in quadrature over terms and
    rows, the systematic ones linearly.  The bound is CONF = 6 times the random scale plus the systematic one.  The
    fp32 rounding of the weights is one shift shared by every row, so its effect is added exactly (the oracle at the
    rounded weights less the oracle at the weights).  Dropping the lo half of the split leaves a random per-term error
    near 2^-11 |t|, about 2^13 / C_TERM = 680 times the term scale here, which the bound rejects (tests/test_mlp_cpu.py
    emulates both products on the CPU).
    """
    params = unpack(layers, w)
    a, z = forward(layers, w, X)
    n = z.shape[0]
    ones = np.ones((n, 1))
    va, sa, vz, sz = _forward_err(params, a, z)
    p = softmax(z)
    yi = np.asarray(y).astype(np.int64)
    rows = np.arange(n)
    mix = (p ** 2 * vz).sum(axis=1, keepdims=True)                      # var of sum_j p_j dz_j
    smix = (p * sz).sum(axis=1, keepdims=True)
    vloss = mix[:, 0] + vz[rows, yi]
    sloss = smix[:, 0] + sz[rows, yi]
    delta = p.copy()
    delta[rows, yi] -= 1.0
    vd = p ** 2 * (vz + mix) + (RHO * delta) ** 2 + TINY ** 2
    sd = p * (sz + smix)
    bF = CONF * math.sqrt(vloss.sum()) / n + sloss.sum() / n
    bounds = [None] * len(params)
    for l in range(len(params) - 1, -1, -1):
        Aa = np.hstack([a[l], ones])                      # [a | 1]: rows x (numIn + 1)
        vAa = np.hstack([va[l], np.zeros((n, 1))])
        sAa = np.hstack([sa[l], np.zeros((n, 1))])
        vp, sp = _product_err(Aa.T, delta.T, unit=512)
        vg = vp + vAa.T @ (delta ** 2) + (Aa ** 2).T @ vd
        sg = sp + sAa.T @ np.abs(delta) + np.abs(Aa).T @ sd
        gb = (CONF * np.sqrt(vg) + sg) / n                # [numIn + 1, numOut]: row i, column o
        bounds[l] = (gb[:-1].T, gb[-1])
        if l > 0:
            Wl = params[l][0]
            back = delta @ Wl
            vp, sp = _product_err(delta, Wl.T)
            vback, sback = vp + vd @ (Wl ** 2), sp + sd @ np.abs(Wl)
            sl = a[l] * (1.0 - a[l])
            dsl = np.abs(1.0 - 2.0 * a[l])
            delta = back * sl
            vd = sl ** 2 * vback + back ** 2 * dsl ** 2 * va[l] + (RHO * delta) ** 2 + TINY ** 2
            sd = sl * sback + np.abs(back) * dsl * sa[l]
    # the device's weights are their fp32 roundings, the same for every row: that shift is systematic, not random, so
    # it is taken exactly (the biases are added in fp64)
    F32, g32 = eval_fg(layers, weights_fp32(layers, w), X, y)
    F0, g0 = eval_fg(layers, w, X, y)
    return bF + abs(F32 - F0), pack(bounds) + np.abs(g32 - g0)


def weights_fp32(layers, w):
    """The weights as the wgmma path uploads them: every W_l entry rounded to fp32, the biases kept in fp64."""
    return pack([(W.astype(np.float32).astype(np.float64), b) for W, b in unpack(layers, w)])


def _tf32(x):
    """Round-to-nearest (ties away) fp32 -> tf32, as rn_tf32_bits does."""
    b = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)
    return ((b + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).view(np.float32)


def _split(x):
    x = np.asarray(x, dtype=np.float32)
    hi = _tf32(x)
    return hi.astype(np.float64), _tf32(x - hi).astype(np.float64)


def _emu_product(A, B, split, unit=None):
    """A [M, K] . B [N, K]^T as k_mlp_wg forms it: per 32-wide chunk the tf32 split products (split = 3: lo.hi + hi.lo
    + hi.hi; split = 1: hi.hi alone) summed and rounded to fp32, chunk sums added in fp32; with `unit`, fp32 sums per
    unit of that many K, added in fp64."""
    Ah, Al = _split(A)
    Bh, Bl = _split(B)
    K = A.shape[1]
    span = unit or K
    total = np.zeros((A.shape[0], B.shape[0]))
    for u in range(0, K, span):
        acc2 = np.zeros((A.shape[0], B.shape[0]), dtype=np.float32)
        for c in range(u, min(K, u + span), 32):
            sl = slice(c, c + 32)
            part = Ah[:, sl] @ Bh[:, sl].T
            if split == 3:
                part = part + Al[:, sl] @ Bh[:, sl].T + Ah[:, sl] @ Bl[:, sl].T
            acc2 = (acc2 + part.astype(np.float32)).astype(np.float32)
        total += acc2
    return total


def emulate_wgmma(layers, w, X, y, split=3):
    """F and the gradient as the wgmma path computes them (split = 3), or with the lo half of the split dropped
    (split = 1): fp32 weights and activations, fp64 bias, softmax and loss, fp32 deltas, 512-row Gram units."""
    params = unpack(layers, w)
    Wf = [W.astype(np.float32) for W, _ in params]
    a = [np.asarray(X, dtype=np.float32)]
    for l, (W, b) in enumerate(params[:-1]):
        zz = _emu_product(a[l], Wf[l], split).astype(np.float32).astype(np.float64) + b
        a.append((1.0 / (1.0 + np.exp(-zz))).astype(np.float32))
    W, b = params[-1]
    z = (_emu_product(a[-1], Wf[-1], split).astype(np.float32).astype(np.float64) + b).astype(np.float32)
    z = z.astype(np.float64)
    n = z.shape[0]
    yi = np.asarray(y).astype(np.int64)
    m = z.max(axis=1, keepdims=True)
    F = float(np.mean(np.log(np.exp(z - m).sum(axis=1)) - (z[np.arange(n), yi] - m[:, 0])))
    delta = softmax(z)
    delta[np.arange(n), yi] -= 1.0
    delta = delta.astype(np.float32)
    grads = [None] * len(params)
    for l in range(len(params) - 1, -1, -1):
        Aa = np.hstack([a[l], np.ones((n, 1), dtype=np.float32)])
        G = _emu_product(Aa.T, delta.T, split, unit=512) / n
        grads[l] = (G[:-1].T, G[-1])
        if l > 0:
            back = _emu_product(delta, Wf[l].T, split).astype(np.float32)
            delta = (back * (a[l] * (np.float32(1.0) - a[l]))).astype(np.float32)
    return F, pack(grads)


def init_weights(layers, seed):
    """The start of b2k_mlp_fit without initialWeights: (u 4.8 - 2.4) / sqrt(numIn), u from splitmix64(seed ^
    splitmix64(j)) >> 11 times 2^-53 over the flat index j."""
    M = (1 << 64) - 1

    def sm64(z):
        z = (z + 0x9E3779B97F4A7C15) & M
        z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M
        z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M
        return z ^ (z >> 31)

    out, j = [], 0
    for i in range(1, len(layers)):
        sc = 1.0 / math.sqrt(layers[i - 1])
        for _ in range(layers[i] * (layers[i - 1] + 1)):
            u = (sm64((seed ^ sm64(j)) & M) >> 11) * 2.0 ** -53
            out.append((u * 4.8 - 2.4) * sc)
            j += 1
    return np.array(out)


def gd(fun, w0, max_iter, tol, step_size):
    """MLlib's full-batch GradientDescent with SimpleUpdater -> (w, history of F at each step's start point)."""
    w = np.array(w0, dtype=np.float64)
    hist = []
    for t in range(1, max_iter + 1):
        F, g = fun(w)
        hist.append(F)
        wn = w - step_size / math.sqrt(t) * g
        done = np.linalg.norm(wn - w) < tol * max(np.linalg.norm(wn), 1.0)
        w = wn
        if done:
            break
    return w, hist


def predict(layers, w, X):
    """rawPrediction z, probability softmax(z), prediction first argmax."""
    _, z = forward(layers, w, X)
    return z, softmax(z), np.argmax(z, axis=1).astype(np.float64)
