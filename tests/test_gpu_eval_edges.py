"""The evaluation passes (b2k_eval.cu) and the curve pass (b2k_binary.cu) against the high-precision oracles of
tests/eval_oracle.py and tests/rf_oracle.py, at the class counts, widths, chunkings and scales where their loops and
branches change.  Nothing here is compared with transform(): that shares b2k_rows.cuh with the passes under test.

Bounds (u = 2^-53; derived as in tests/test_gpu_linreg.py, from the number of roundings on each path):
  margins     b + x . w_k on the device is d + 1 fp64 FMAs / adds in a lane-split order: within
              beta = (d + 1) 2^-52 (sum_j |x_j w_kj| + |b_k|) of the exact value (eval_oracle.linear_margins).  The data
              have no row whose predicted class beta leaves open, so every count is exact.
  log-loss    a row's -log p_y moves by at most 2 max_k beta_k through its margins (the gradient of log-sum-exp has
              1-norm <= 2), plus the finish: the exps, the K-term denominator, the divide and the log round
              (K + 8) 2^-52 (1 + max_k |m_k - m_max|) + 2^-52 (-log p_y); a binomial 1 - p1 adds 2^-52 / p_y.  The
              device sums the rows in chains of at most D = ceil(TR / 32) + 5 + ceil(tiles / grid) + grid additions
              (lane stride, butterfly, tiles of one CTA, the CTA fold): D u sum(-log p_y) more.  Forests form p_y with
              the oracle's bits, so only the log and the sum remain.
  moments     count exact.  With values v (off by at most Delta per row: beta for an identity prediction, 0 for a
              forest's), E = 4 D u max|v| for the error of a mean formed by tile sums and Chan merges along a chain of
              D, A = sum |v - mean| and Q = m2n: mean within Delta + E; m2n within 2 (2 A (2 Delta + 4 E) +
              2 (D + 4) u Q + n (2 Delta + E)^2); m2 within 2 sum|v| Delta + n Delta^2 + (D + 1) u sum v^2; l1 within
              n Delta + D u sum|v|.
  curve       every trapezoid is >= 0 and formed with the oracle's operations; the device adds them in chains of at
              most per / 256 + 8 + 1056 (a thread's segments, the block tree, the fold over <= 8 CTAs per SM), so the
              area holds 1e-12 relative at n < 2^31.
"""
import math

import numpy as np
import pytest
import torch

import eval_oracle as eo
import rf_oracle
from spark_rapids_ml_b200 import _native

pytestmark = pytest.mark.gpu
U = 2.0 ** -53
NAMES = ("areaUnderROC", "areaUnderPR")

# b2k_eval.cu's tiling constants, restated to predict tiles, chunks and the shared-memory limit
EV_NT, EV_NW, EV_MAX_ROWS, EV_MAX_CHUNK, NREG = 256, 8, 256, 32, 15
EV_TILE_BYTES, EV_FTILE_BYTES, EV_SMEM_MAX = 16384, 32768, 100 * 1024


def row_lanes(d):
    L = 1
    while L < 32 and 4 * L < d:
        L <<= 1
    return L


def tile_rows(dpad, step, tile_bytes):
    tr = min(EV_MAX_ROWS, max(1, tile_bytes // (dpad * 4)))
    return tr // step * step if tr >= step else tr


def lin_tile(d):
    dpad = (d + 3) & ~3
    return dpad, tile_rows(dpad, EV_NW * (32 // row_lanes(d)), EV_TILE_BYTES)


def forest_tile(d):
    dpad = (d + 3) & ~3
    return dpad, tile_rows(dpad, 1, EV_FTILE_BYTES)


def ev_carve(TR, dpad, m, C, cls):
    """Bytes of ev_carve: each region rounded up to 16 bytes."""
    r16 = lambda b: (b + 15) & ~15   # noqa: E731
    return (r16(TR * dpad * 4) + r16(TR * 4) + r16(m * TR * 8) + r16(C * 4 if cls else 0)
            + r16(m * 2 * C * 4 if cls else 0) + r16(m * (1 if cls else NREG) * 8))


def n_chunks(m, TR, dpad, C, cls):
    """chunk_end's rule: the longest prefix under EV_SMEM_MAX, at most EV_MAX_CHUNK models."""
    first, k = 0, 0
    while first < m:
        e = first + 1
        while e < m and e - first < EV_MAX_CHUNK and ev_carve(TR, dpad, e + 1 - first, C, cls) <= EV_SMEM_MAX:
            e += 1
        first, k = e, k + 1
    return k


def depth(n, TR, limit=0):
    """The longest chain of additions from a row's value to a folded sum (see the header)."""
    tiles = -(-n // TR)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    grid = max(1, min(tiles, 2 * sms, limit) if limit else min(tiles, 2 * sms))
    return -(-TR // 32) + 5 + -(-tiles // grid) + grid


@pytest.fixture(scope="module")
def ctx():
    with _native.Context(0) as c:
        yield c


@pytest.fixture
def grid_limit(ctx):
    def set_(g):
        ctx.set_option("grid_limit", g)
    yield set_
    ctx.set_option("grid_limit", 0)


def _dev(*a):
    return [torch.from_numpy(np.ascontiguousarray(v)).cuda() for v in a]


# ---- linear classification ----
def _softmax_model(rng, K, d, class_values=None, scale=2.0):
    W = rng.normal(size=(K, d)) * scale / math.sqrt(d)
    return {"kind": "softmax", "W": W, "b": rng.normal(size=K),
            "class_values": np.arange(K, dtype=np.float64) if class_values is None else class_values}


def _binomial_model(rng, d, class_values=(0.0, 1.0)):
    return {"kind": "logistic", "W": rng.normal(size=(1, d)) * 2.0 / math.sqrt(d), "b": rng.normal(size=1),
            "class_values": np.asarray(class_values, dtype=np.float64)}


def _linear_oracle(X, y, md, C, D, eps=1e-15):
    """The accumulators of one linear classifier and the bound on its loss (header)."""
    m, beta, unsettled = eo.linear_margins(X, md["W"], md["b"], binomial=md["kind"] == "logistic")
    assert unsettled.size == 0, f"{unsettled.size} rows with an unsettled class"
    pred, probs = eo.linear_predictions(m, md["kind"], md["class_values"])
    py = eo.label_prob(probs, y)
    acc = eo.classification_acc(y, pred, py, C, eps)
    pyf = py.astype(np.float64)
    inside = pyf > 0
    assert not np.any(inside & (pyf > 0.5 * eps) & (pyf < 2 * eps)), "a p_y at the eps clip"
    ell = -np.log(np.maximum(pyf, eps))
    K = m.shape[1]
    if md["kind"] == "logistic":
        per = beta[:, 0] + 9 * 2.0 ** -52 * (1 + np.abs(m[:, 0])) + np.where(inside, 2.0 ** -52 / np.maximum(pyf, eps), 0)
    else:
        per = 2 * beta.max(axis=1) + (K + 8) * 2.0 ** -52 * (1 + (m.max(axis=1) - m.min(axis=1)))
    acc["loss_bound"] = float(np.sum(per + 2.0 ** -52 * ell) + D * U * np.sum(ell))
    return acc


def _check_linear(ctx, X, y, models, got=None):
    n, d = X.shape
    if got is None:
        got = ctx.eval_linear(*_dev(X, y), models)
    C = got["label_count"].size
    D = depth(n, lin_tile(d)[1])
    assert got["n"] == n
    np.testing.assert_array_equal(got["label_count"], np.bincount(y.astype(np.int64), minlength=C))
    for i, md in enumerate(models):
        want = _linear_oracle(X, y, md, C, D)
        np.testing.assert_array_equal(got["tp"][i], want["tp"], err_msg=f"tp of model {i}")
        np.testing.assert_array_equal(got["fp"][i], want["fp"], err_msg=f"fp of model {i}")
        assert abs(got["loss"][i] - want["loss"]) <= want["loss_bound"], (i, got["loss"][i], want["loss"])
    return got


def _cls_data(rng, n, d, top):
    X = rng.normal(size=(n, d)).astype(np.float32)
    y = rng.integers(0, top + 1, n).astype(np.float32)
    y[0] = top
    return X, y


@pytest.mark.parametrize("K", [7, 8, 9, 16, 17, 100])
def test_softmax_class_chunks(ctx, K):
    """k_eval_linear's loop over chunks of EV_RC = 8 classes: K = 7, 8 (one chunk, full or not), 9, 16, 17 (a second and
    third chunk, a one-class remainder) and 100 (13 chunks); labels up to K + 2 take the p_y = 0 branch.  Counts exact,
    loss within the margin / finish / summation bound of the header."""
    rng = np.random.default_rng(K)
    X, y = _cls_data(rng, 2000, 33, K + 2)
    _check_linear(ctx, X, y, [_softmax_model(rng, K, 33), _softmax_model(rng, K, 33)])


@pytest.mark.parametrize("d", [1, 3, 4, 5, 124, 125, 513, 1024])
def test_widths(ctx, d):
    """Lanes per row L = 1 .. 32 (d = 1 .. 1024 = B2K_LOGREG_MAX_D), the scalar staging path (d % 4 != 0) and the float4
    one, tiles of fewer rows than a step from d = 513; K = 9 (two class chunks) beside a binomial model with class values
    [3, 7].  Counts exact, loss within the header's bound."""
    rng = np.random.default_rng(100 + d)
    X, y = _cls_data(rng, 1500, d, 10)
    _check_linear(ctx, X, y, [_softmax_model(rng, 9, d), _binomial_model(rng, d, (3.0, 7.0))])


def test_mixed_kinds_share_margin_slots(ctx):
    """One chunk of binomial and softmax models of K = 3, 17, 2, 9: the margin slots sized for K = 17 are reused by
    every softmax model in turn, the binomial margin stays in a register; labels up to 19 (past every model)."""
    rng = np.random.default_rng(7)
    d = 24
    X, y = _cls_data(rng, 3001, d, 19)
    models = [_binomial_model(rng, d), _softmax_model(rng, 3, d), _softmax_model(rng, 17, d),
              _binomial_model(rng, d, (3.0, 7.0)), _softmax_model(rng, 2, d), _softmax_model(rng, 9, d)]
    _check_linear(ctx, X, y, models)


def test_linear_shared_memory_chunks(ctx):
    """C = 1024 (labels up to 1023) and M = 40: each model's tp / fp counters take 8 KB, so chunk_end splits at
    EV_SMEM_MAX well below the 32-model cap (asserted through the launch count).  Counts exact, loss within the header's
    bound, and every model bitwise equal to itself evaluated alone."""
    rng = np.random.default_rng(11)
    n, d, M = 3000, 33, 40
    models = [_softmax_model(rng, int(rng.integers(2, 6)), d) for _ in range(M)]
    for md in models:
        md["class_values"] = rng.choice(1024, md["W"].shape[0], replace=False).astype(np.float64)
    pool = np.concatenate([md["class_values"] for md in models])
    X = rng.normal(size=(n, d)).astype(np.float32)
    y = np.where(rng.random(n) < 0.5, rng.choice(pool, n), rng.integers(0, 1024, n)).astype(np.float32)
    y[0] = 1023
    dpad, TR = lin_tile(d)
    chunks = n_chunks(M, TR, dpad, 1024, True)
    assert chunks > -(-M // EV_MAX_CHUNK)
    ctx.reset_stats()
    got = ctx.eval_linear(*_dev(X, y), models)
    assert ctx.stats()["kernel_launches"] == 1 + 2 * chunks   # the label check, then a pass and a fold per chunk
    _check_linear(ctx, X, y, models, got)
    Xd, yd = _dev(X, y)
    for i, md in enumerate(models):
        one = ctx.eval_linear(Xd, yd, [md])
        assert one["loss"][0].tobytes() == got["loss"][i].tobytes(), i
        np.testing.assert_array_equal(one["tp"][0], got["tp"][i])
        np.testing.assert_array_equal(one["fp"][0], got["fp"][i])


# ---- forests ----
def _forest(rng, d, T, dep, V, regression=False, root_feature=None):
    """T complete trees of depth dep in rf_fit's layout (breadth-first, tree-local children, a value row per node);
    every root splits on root_feature (default d - 1, the last staged column)."""
    feat, thr, ch, val, off = [], [], [], [], [0]
    nin, nn = 2 ** dep - 1, 2 ** (dep + 1) - 1
    for _ in range(T):
        for i in range(nn):
            if i < nin:
                feat.append((d - 1 if root_feature is None else root_feature) if i == 0 else int(rng.integers(0, d)))
                thr.append(float(rng.normal() * 0.7))
                ch.append((2 * i + 1, 2 * i + 2))
            else:
                feat.append(-1)
                thr.append(0.0)
                ch.append((-1, -1))
            val.append(rng.normal(size=1) if regression else rng.dirichlet(np.ones(V) * 0.5))
        off.append(off[-1] + nn)
    V = 1 if regression else V
    return {"tree_offsets": np.array(off, np.int64), "feature": np.array(feat, np.int32),
            "threshold": np.array(thr, np.float32), "children": np.array(ch, np.int32).reshape(-1, 2),
            "value": np.array(val, np.float64).reshape(-1, V), "n_values": V}


def _check_forest_cls(ctx, X, y, forests, got=None, limit=0):
    n, d = X.shape
    if got is None:
        got = ctx.eval_forest(*_dev(X, y), forests, True)
    C = got["label_count"].size
    D = depth(n, forest_tile(d)[1], limit)
    np.testing.assert_array_equal(got["label_count"], np.bincount(y.astype(np.int64), minlength=C))
    for i, f in enumerate(forests):
        raw, prob, pred = rf_oracle.predict(X, f, True)
        py = eo.label_prob(prob, y)
        want = eo.classification_acc(y, pred, py, C)
        ell = -np.log(np.maximum(py, 1e-15))
        bound = 2.0 ** -51 * ell.sum() + D * U * ell.sum()
        np.testing.assert_array_equal(got["tp"][i], want["tp"], err_msg=f"tp of forest {i}")
        np.testing.assert_array_equal(got["fp"][i], want["fp"], err_msg=f"fp of forest {i}")
        assert abs(got["loss"][i] - want["loss"]) <= bound, (i, got["loss"][i], want["loss"])
    return got


def _moment_bounds(R, v_abs_max, v_abs_sum, v_sq_sum, A, n, delta, D):
    E = 4 * D * U * v_abs_max
    return np.array([0.0, delta + E, 2 * (2 * A * (2 * delta + 4 * E) + 2 * (D + 4) * U * R[2] + n * (2 * delta + E) ** 2),
                     2 * v_abs_sum * delta + n * delta ** 2 + (D + 1) * U * v_sq_sum, n * delta + D * U * v_abs_sum])


def _moment_oracle(y, pred):
    """regression_acc of (y, pred) and, per column, (max|v|, sum|v|, sum v^2, sum|v - mean|) for the bounds."""
    want = eo.regression_acc(y, pred)
    yy = y.astype(np.float64)
    scale = [(float(np.abs(v).max()), float(np.abs(v).sum()), float((v * v).sum()), float(np.abs(v - want[c][1]).sum()))
             for c, v in enumerate((yy, yy - pred, pred))]
    return want, scale, y.size


def _check_moments(got, oracle, delta, D, label=""):
    """got [3, 5] against the oracle within the header's moment bounds; delta [3] per column."""
    want, scale, n = oracle
    for c in range(3):
        b = _moment_bounds(want[c], *scale[c], n, delta[c], D)
        assert got[c][0] == want[c][0], (label, c)
        err = np.abs(got[c] - want[c])
        assert np.all(err <= b), (label, c, err.tolist(), b.tolist())


def _check_forest_reg(ctx, X, y, forests, got=None, limit=0, oracles=None):
    n, d = X.shape
    if got is None:
        got = ctx.eval_forest(*_dev(X, y), forests, False)
    D = depth(n, forest_tile(d)[1], limit)
    for i, f in enumerate(forests):
        oracle = oracles[i] if oracles else _moment_oracle(y, rf_oracle.predict(X, f, False)[2])
        _check_moments(got["reg"][i], oracle, (0.0, 0.0, 0.0), D, f"forest {i}")
    return got


@pytest.mark.parametrize("d", [80, 300])
def test_forest_partial_thread_groups(ctx, d):
    """TR = 102 (d = 80: two groups of 102 threads, 52 idle) and TR = 27 (d = 300: nine groups, 13 idle), 20 forests so
    each group walks several; classification with labels up to V + 2 (p_y = 0 past V) and regression.  Per-row
    predictions are rf_oracle.predict's bits: counts exact, loss and moments within the header's bounds."""
    assert forest_tile(d)[1] == {80: 102, 300: 27}[d]
    rng = np.random.default_rng(d)
    n = 2503
    X = rng.normal(size=(n, d)).astype(np.float32)
    y = rng.integers(0, 6, n).astype(np.float32)
    _check_forest_cls(ctx, X, y, [_forest(rng, d, 3, 4, 4) for _ in range(20)])
    yr = rng.normal(size=n).astype(np.float32)
    _check_forest_reg(ctx, X, yr, [_forest(rng, d, 3, 4, 1, regression=True) for _ in range(20)])


def test_forest_one_row_tiles(ctx):
    """d = 5000: TR = 1, 256 groups of one thread, one row per tile and 33 forests in two chunks (the 32-model cap).  A
    chunk holds at most 32 forests, so here every forest has a group of its own; test_forest_partial_thread_groups runs
    more forests than groups.  Counts exact, loss within the header's bound."""
    d = 5000
    assert forest_tile(d)[1] == 1
    rng = np.random.default_rng(5000)
    n = 300
    X = rng.normal(size=(n, d)).astype(np.float32)
    y = rng.integers(0, 4, n).astype(np.float32)
    forests = [_forest(rng, d, 2, 3, 3) for _ in range(33)]
    ctx.reset_stats()
    got = ctx.eval_forest(*_dev(X, y), forests, True)
    assert ctx.stats()["kernel_launches"] == 1 + 2 * 2
    _check_forest_cls(ctx, X, y, forests, got)


@pytest.mark.parametrize("classification", [False, True])
def test_forest_width_limit(ctx, classification):
    """The largest d whose one-row tile fits EV_SMEM_MAX (ev_carve's rule) evaluates, with every root splitting on
    feature d - 1; the next multiple of 4 fails at the host check with B2K_ERR_UNSUPPORTED (code 4) and the documented
    message, before any pass runs."""
    C = 2 if classification else 0
    d = max(dp for dp in range(24000, 26000, 4) if ev_carve(1, dp, 1, C, classification) <= EV_SMEM_MAX)
    assert forest_tile(d)[1] == 1
    rng = np.random.default_rng(d)
    n = 40
    X = rng.normal(size=(n, d)).astype(np.float32)
    if classification:
        y = rng.integers(0, 2, n).astype(np.float32)
        _check_forest_cls(ctx, X, y, [_forest(rng, d, 2, 2, 2)])
    else:
        y = rng.normal(size=n).astype(np.float32)
        _check_forest_reg(ctx, X, y, [_forest(rng, d, 2, 2, 1, regression=True)])
    d2 = d + 4
    X2 = rng.normal(size=(n, d2)).astype(np.float32)
    f = _forest(rng, d2, 1, 2, 2 if classification else 1, regression=not classification)
    with pytest.raises(_native.B2KError, match=f"evaluation: one forest needs {ev_carve(1, d2, 1, C, classification)} "
                                               f"bytes of shared memory, above {EV_SMEM_MAX}") as e:
        ctx.eval_forest(*_dev(X2, y), [f], classification)
    assert e.value.code == 4


def test_forest_split_past_d_is_refused(ctx):
    """A node splitting on feature d (one past the staged columns) is refused by the host table check."""
    rng = np.random.default_rng(1)
    X = rng.normal(size=(50, 7)).astype(np.float32)
    y = rng.integers(0, 2, 50).astype(np.float32)
    bad = _forest(rng, 7, 1, 2, 2, root_feature=7)
    with pytest.raises(_native.B2KError, match="b2k_eval_forest: a node splits on feature 7 >= d = 7"):
        ctx.eval_forest(*_dev(X, y), [bad], True)
    scores, pos = ctx.binary_buffers(1, 50)
    with pytest.raises(_native.B2KError, match="b2k_eval_forest_scores: a node splits on feature 7 >= d = 7"):
        ctx.binary_scores_forest(*_dev(X, y), [bad], scores, pos)


@pytest.mark.parametrize("V,top", [(2, 5), (64, 70)])
def test_forest_values_and_labels(ctx, V, top):
    """V = 2 forests scored on labels up to 5 (p_y = 0 for labels 2 .. 5; C from the labels), and V = 64 (C from the
    forests' values and labels up to 70).  Counts exact, loss within the header's bound."""
    rng = np.random.default_rng(V)
    n, d = 4001, 12
    X = rng.normal(size=(n, d)).astype(np.float32)
    y = rng.integers(0, top + 1, n).astype(np.float32)
    got = _check_forest_cls(ctx, X, y, [_forest(rng, d, 4, 5, V) for _ in range(3)])
    assert got["label_count"].size == max(V, top + 1)


def test_forest_shared_memory_chunks(ctx):
    """C = 1024 and M = 40 forests: chunk_end splits at EV_SMEM_MAX below the 32-model cap (launch count); counts exact,
    loss within the header's bound, each forest bitwise equal to itself evaluated alone."""
    rng = np.random.default_rng(12)
    n, d, M = 3000, 8, 40
    X = rng.normal(size=(n, d)).astype(np.float32)
    y = np.where(rng.random(n) < 0.7, rng.integers(0, 3, n), rng.integers(0, 1024, n)).astype(np.float32)
    y[0] = 1023
    forests = [_forest(rng, d, 2, 4, 3) for _ in range(M)]
    dpad, TR = forest_tile(d)
    chunks = n_chunks(M, TR, dpad, 1024, True)
    assert chunks > -(-M // EV_MAX_CHUNK)
    ctx.reset_stats()
    got = ctx.eval_forest(*_dev(X, y), forests, True)
    assert ctx.stats()["kernel_launches"] == 1 + 2 * chunks
    _check_forest_cls(ctx, X, y, forests, got)
    Xd, yd = _dev(X, y)
    for i, f in enumerate(forests):
        one = ctx.eval_forest(Xd, yd, [f], True)
        assert one["loss"][0].tobytes() == got["loss"][i].tobytes(), i
        np.testing.assert_array_equal(one["tp"][0], got["tp"][i])
        np.testing.assert_array_equal(one["fp"][0], got["fp"][i])


# ---- regression at scale ----
@pytest.mark.parametrize("offset,scale", [(1e6, 1.0), (0.0, 1e-6)])
def test_identity_moments_at_scale(ctx, grid_limit, offset, scale):
    """n = 3 000 017 rows, d = 8, two identity models, at the default grid (about 44 tiles per CTA) and at grid_limit = 3
    (about 3 900 tiles per CTA, the long Chan chains); labels at an offset of 1e6, or scaled by 1e-6.  Count exact, the
    other moments within the header's bounds with Delta = beta for the prediction columns."""
    rng = np.random.default_rng(int(offset) + 3)
    n, d = 3_000_017, 8
    X = rng.normal(size=(n, d)).astype(np.float32)
    w = rng.normal(size=d)
    y = ((offset + X.astype(np.float64) @ w + rng.normal(size=n)) * scale).astype(np.float32)
    models = [{"kind": "identity", "W": ((w + 0.1 * rng.normal(size=d)) * scale)[None, :],
               "b": np.array([(offset + 0.3 * i) * scale])} for i in range(2)]
    oracle = []
    for md in models:
        m, beta, _ = eo.linear_margins(X, md["W"], md["b"])
        p, bmax = m[:, 0], float(beta.max())
        # the residual y - p is rounded once on each side: beta + 2 u max|v| apart
        oracle.append((_moment_oracle(y, p), (0.0, bmax + 2 * U * float(np.abs(y).max() + np.abs(p).max()), bmax)))
    Xd, yd = _dev(X, y)
    TR = lin_tile(d)[1]
    for limit in (0, 3):
        grid_limit(limit)
        got = ctx.eval_linear(Xd, yd, models)
        D = depth(n, TR, limit)
        for i, (orc, delta) in enumerate(oracle):
            _check_moments(got["reg"][i], orc, delta, D, f"model {i} grid_limit {limit}")


@pytest.mark.parametrize("offset,scale", [(1e6, 1.0), (0.0, 1e-6)])
def test_forest_moments_at_scale(ctx, grid_limit, offset, scale):
    """n = 1 000 003 rows, three regression forests whose leaves sit at the label's offset / scale, at the default grid
    and at grid_limit = 3.  Predictions are rf_oracle.predict's bits (Delta = 0): count exact, the other moments within
    the header's bounds."""
    rng = np.random.default_rng(int(offset) + 4)
    n, d = 1_000_003, 8
    X = rng.normal(size=(n, d)).astype(np.float32)
    y = ((offset + X[:, 0].astype(np.float64) + rng.normal(size=n)) * scale).astype(np.float32)
    forests = []
    for _ in range(3):
        f = _forest(rng, d, 4, 5, 1, regression=True)
        f["value"] = (offset + f["value"]) * scale
        forests.append(f)
    oracles = [_moment_oracle(y, rf_oracle.predict(X, f, False)[2]) for f in forests]
    Xd, yd = _dev(X, y)
    for limit in (0, 3):
        grid_limit(limit)
        _check_forest_reg(ctx, X, y, forests, ctx.eval_forest(Xd, yd, forests, False), limit, oracles)


# ---- score passes ----
@pytest.mark.parametrize("d", [1, 5, 128, 1024])
def test_linear_scores(ctx, grid_limit, d):
    """k_score_linear for softmax K = 2, 9, 17, 100 and a binomial model in one pass: each score within beta of the
    oracle's class-1 margin, and bitwise equal to rawPrediction[:, 1] of logreg_predict (k_logreg_rows, chunks of 8
    classes) -- class 1's FMA chain does not depend on the chunk width.  grid_limit 1 and 3 give the default grid's bits;
    pos = y > 0.5 at 0.5, nextafter(0.5f) and -1."""
    rng = np.random.default_rng(200 + d)
    n = 6000 if d <= 128 else 1500
    X = rng.normal(size=(n, d)).astype(np.float32)
    y = rng.integers(0, 2, n).astype(np.float32)
    y[:3] = [0.5, np.nextafter(np.float32(0.5), np.float32(1)), -1.0]
    models = [_softmax_model(rng, K, d) for K in (2, 9, 17, 100)] + [_binomial_model(rng, d)]
    Xd, yd = _dev(X, y)
    scores, pos = ctx.binary_buffers(len(models), n)
    ctx.binary_scores_linear(Xd, yd, models, scores, pos)
    s = scores.cpu().numpy().copy()
    np.testing.assert_array_equal(pos.cpu().numpy(), (y > 0.5).astype(np.uint8))
    assert pos.cpu().numpy()[:3].tolist() == [0, 1, 0]
    for i, md in enumerate(models):
        m, beta, _ = eo.linear_margins(X, md["W"], md["b"])
        c = 0 if md["kind"] == "logistic" else 1
        assert np.all(np.abs(s[i] - m[:, c]) <= beta[:, c]), i
        raw, _, _ = ctx.logreg_predict(Xd, md["W"], md["b"], md["class_values"])
        assert s[i].tobytes() == raw[:, 1].cpu().numpy().tobytes(), i
    for limit in (1, 3):
        grid_limit(limit)
        ctx.binary_scores_linear(Xd, yd, models, scores, pos)
        assert scores.cpu().numpy().tobytes() == s.tobytes(), limit


@pytest.mark.parametrize("d", [5, 80, 300])
def test_forest_scores(ctx, grid_limit, d):
    """k_score_forest at TR = 256, 102 and 27 with 12 forests (more than the groups at d = 80 and 300): bitwise equal to
    rf_oracle.predict's raw[:, 1]; grid_limit 1 and 3 give the default grid's bits."""
    rng = np.random.default_rng(300 + d)
    n = 5003
    X = rng.normal(size=(n, d)).astype(np.float32)
    y = rng.integers(0, 2, n).astype(np.float32)
    forests = [_forest(rng, d, 3, 4, int(rng.integers(2, 5))) for _ in range(12)]
    Xd, yd = _dev(X, y)
    scores, pos = ctx.binary_buffers(len(forests), n)
    ctx.binary_scores_forest(Xd, yd, forests, scores, pos)
    s = scores.cpu().numpy().copy()
    for i, f in enumerate(forests):
        raw, _, _ = rf_oracle.predict(X, f, True)
        assert s[i].tobytes() == np.ascontiguousarray(raw[:, 1]).tobytes(), i
    for limit in (1, 3):
        grid_limit(limit)
        ctx.binary_scores_forest(Xd, yd, forests, scores, pos)
        assert scores.cpu().numpy().tobytes() == s.tobytes(), limit


# ---- the curve pass ----
def _kinds(rng, n):
    return np.stack([rng.normal(size=n), np.round(rng.normal(size=n), 3), rng.choice([-0.5, 2.0], size=n),
                     np.full(n, 0.25)])


def _label_sets(n):
    alt = (np.arange(n) % 2).astype(np.float64)
    one = np.zeros(n)
    one[n // 2] = 1.0
    return {"alternating": alt, "one_positive": one, "all_but_one": 1.0 - one}


def _close(got, want):
    return abs(got - want) <= 1e-12 * abs(want)


@pytest.mark.parametrize("n", [1, 2, 255, 256, 257, 65_537, 4_000_037])
def test_curve_at_scale(ctx, n):
    """k_bin_area over 1 .. 8 x SMs CTAs (the grid cap from n = 270 337 on an H100) and, at n = 4 000 037, about 15
    segments per thread (the multi-trip loop); continuous, 3-decimal, two-valued and constant scores; numBins 0, 1, 7,
    1000, D / 2, D - 1, D + 5; alternating, single-positive and all-but-one-positive labels.  Both metrics within
    1e-12 relative of the fsum oracle (header: chains of at most per / 256 + 8 + 1056 non-negative terms)."""
    rng = np.random.default_rng(n)
    S = _kinds(rng, n)
    Sd = torch.from_numpy(S).cuda()
    for lname, y in _label_sets(n).items():
        pos = torch.from_numpy((y > 0.5).astype(np.uint8)).cuda()
        counts = [eo.binary_counts(S[k], y) for k in range(S.shape[0])]
        memo = {}

        def want(k, bins, name):   # the area depends on numBins through the group size alone
            p, q = counts[k]
            g = p.size // bins if bins else 1
            key = (k, g if g >= 2 else 1, name)
            if key not in memo:
                memo[key] = eo.binary_area(p, q, name, bins)
            return memo[key]

        for bins in (0, 1, 7, 1000):
            for name in NAMES:
                got = ctx.eval_binary(Sd, pos, bins, name)
                for k in range(S.shape[0]):
                    assert _close(got[k], want(k, bins, name)), (lname, k, bins, name, got[k], want(k, bins, name))
        for k, (p, _) in enumerate(counts):
            D = p.size
            for bins in sorted({D // 2, max(D - 1, 0), D + 5} - {0, 1, 7, 1000}):
                for name in NAMES:
                    got = ctx.eval_binary(Sd[k:k + 1].contiguous(), pos, bins, name)[0]
                    assert _close(got, want(k, bins, name)), (lname, k, bins, name, got, want(k, bins, name))


def test_curve_many_models(ctx):
    """M = 130 models at n = 10 000: k_bin_fold's second block of 128 threads; every model against the oracle and
    bitwise equal to itself evaluated alone."""
    rng = np.random.default_rng(130)
    n, M = 10_000, 130
    S = np.round(rng.normal(size=(M, n)) * rng.uniform(0.5, 3.0, size=(M, 1)), int(rng.integers(1, 4)))
    y = rng.integers(0, 2, n).astype(np.float64)
    Sd = torch.from_numpy(S).cuda()
    pos = torch.from_numpy((y > 0.5).astype(np.uint8)).cuda()
    for name in NAMES:
        got = ctx.eval_binary(Sd, pos, 1000, name)
        for i in range(M):
            p, q = eo.binary_counts(S[i], y)
            assert _close(got[i], eo.binary_area(p, q, name, 1000)), (name, i)
            alone = ctx.eval_binary(Sd[i:i + 1].contiguous(), pos, 1000, name)
            assert alone[0].tobytes() == got[i].tobytes(), (name, i)


def test_curve_repeatable_at_scale(ctx):
    """Two calls at n = 4 000 037 (1 056 CTAs on an H100, no atomics) give the same bits."""
    rng = np.random.default_rng(4)
    n = 4_000_037
    Sd = torch.from_numpy(np.stack([rng.normal(size=n), np.round(rng.normal(size=n), 2)])).cuda()
    pos = torch.from_numpy(rng.integers(0, 2, n).astype(np.uint8)).cuda()
    for name in NAMES:
        a = ctx.eval_binary(Sd, pos, 1000, name)
        b = ctx.eval_binary(Sd, pos, 1000, name)
        assert a.tobytes() == b.tobytes(), name
