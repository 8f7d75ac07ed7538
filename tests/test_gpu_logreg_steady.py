"""Logistic regression's device passes in steady state, against the fp64 oracle of tests/logreg_oracle.py.

test_gpu_logreg.py runs every pass at shapes where each CTA sees one tile, the generic pass one chunk, the label pass
a handful of spans and the transform kernel one sweep of its grid.  Here each pass runs past those edges:

- the fused pass (k_logreg_eval) with hundreds of tiles per CTA (option `grid_limit` at n = 20011) and with at least 5
  tiles per CTA at the default grid, for every <KB, NIT> instantiation at its largest d, at ragged K' and tiny d, and on
  each side of every change of its tile height; also where its coverage stops;
- the generic pass over several 64 MB chunks of residuals, with a ragged last chunk;
- rows whose label is none of the classes, and an X that is not 16-byte aligned;
- the label pass at its span cap, with every class value, a count above 2^24 and bad values in its last row;
- the transform kernel (k_logreg_rows in predict mode) and k_linreg_predict over several sweeps of their grids;
- one fit at a capped grid on both paths.

The planner of csrc/b2k_logreg.cu is restated below; each test derives its row counts and the path it expects from it
and the device's SM count and opt-in shared memory, read from torch.
"""
import contextlib

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import logreg_oracle as lo  # noqa: E402
from spark_rapids_ml_b200 import _native  # noqa: E402

N = 20011                     # many tiles at every tile height, a ragged last one
GRID_LIMITS = (1, 3, 7)       # 3 and 7 give the CTAs unequal spans
MIN_TILES_PER_CTA = 5         # at the default grid
MAX_CTAS_PER_SM = 8           # a 256-thread CTA: at most 2048 threads per SM
DEFAULTS = {"kernel_path": 0, "grid_limit": 0}
U = 2.0 ** -53

# ---------------------------------------------------------------------------------------------------------------------
# the planner of csrc/b2k_logreg.cu
# ---------------------------------------------------------------------------------------------------------------------
LR_THREADS = 256
MAX_D = 1024
MAX_CLASSES = 1024
CHUNK_BYTES = 64 << 20        # the generic pass's residual chunk
LABEL_SPAN_ROWS = 1024
RC = 8                        # classes per pass of the transform kernel's k0 loop


def _cdiv(a, b):
    return -(-a // b)


def _sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _smem_optin():
    return torch.cuda.get_device_properties(0).shared_memory_per_block_optin


def tile_stride(d):
    return d + 2 if d & 1 else d + 1


def tile_rows(d):
    return 64 if d <= 128 else 32 if d <= 256 else 16 if d <= 512 else 8


def fused_pick(d, kp):
    """(KB, NIT) of the instantiation K' maps to, or None where its accumulators do not cover d"""
    KB, NIT = (1, 4) if kp <= 1 else (2, 4) if kp <= 2 else (4, 4) if kp <= 4 else (8, 2) if kp <= 8 else (16, 1)
    if d > MAX_D or d * _cdiv(kp, KB) > LR_THREADS * NIT:
        return None
    return KB, NIT


def fused_shape(d, kp, KB, tr):
    nkb = _cdiv(kp, KB)
    parts = LR_THREADS // tr
    fs_n = 1 if nkb >= parts else parts // nkb
    items = d * nkb
    rg = 1 if items >= LR_THREADS else min(tr, LR_THREADS // items)
    return {"nkb": nkb, "parts": parts, "fs_n": fs_n, "items": items, "rg": rg}


def fused_smem(d, kp, KB):
    tr = tile_rows(d)
    f = fused_shape(d, kp, KB, tr)
    dbl = kp * d + kp + f["fs_n"] * tr * kp + 2 * tr * kp + tr
    return dbl * 8 + 2 * tr * tile_stride(d) * 4


def fused_covers(d, kp):
    p = fused_pick(d, kp)
    return p is not None and fused_smem(d, kp, p[0]) <= _smem_optin()


def fused_spans(n, d, cap):
    """(rows per CTA span, CTAs) of the fused grid when at most `cap` CTAs run"""
    tr = tile_rows(d)
    tiles = max(1, _cdiv(n, tr))
    g0 = min(tiles, cap)
    span_rows = _cdiv(tiles, g0) * tr
    return span_rows, max(1, _cdiv(n, span_rows))


def generic_chunk(n, kp):
    return max(1, min(max(n, 1), CHUNK_BYTES // (8 * (kp + 1))))


def label_spans(n):
    """(spans, rows per span) of k_logreg_labels"""
    spans = max(1, min(4 * _sm_count(), _cdiv(n, LABEL_SPAN_ROWS)))
    return spans, max(1, _cdiv(n, spans))


def row_lanes(d):
    L = 1
    while L < 32 and 4 * L < d:
        L <<= 1
    return L


def predict_sweep(d):
    """rows one grid-stride sweep of the transform kernel covers at its grid cap of 8 CTAs per SM; k_linreg_predict
    (256 threads, the same lanes per row) covers at most as many"""
    return 8 * _sm_count() * (LR_THREADS // 32) * (32 // row_lanes(d))


# ---------------------------------------------------------------------------------------------------------------------
# harness
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def ctx():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    with _native.Context(0) as c:
        yield c


@contextlib.contextmanager
def _options(ctx, **kw):
    try:
        for key, v in kw.items():
            ctx.set_option(key, v)
        yield
    finally:
        for key in kw:
            ctx.set_option(key, DEFAULTS[key])


def _case(n, d, kp, seed, offset=0.0, wscale=1.0, margin=None):
    """rows, labels uniform over max(kp, 2) classes 0, 1, ..., and W, b; margin = c: W = +-c / sqrt(d), margins of
    order +-c"""
    rng = np.random.default_rng(seed)
    K = max(kp, 2)
    X = rng.standard_normal(size=(n, d), dtype=np.float32)
    if offset:
        X += np.float32(offset)
    y = rng.integers(0, K, size=n).astype(np.float32)
    W = rng.normal(size=(kp, d)) * wscale / np.sqrt(d)
    if margin is not None:
        W = np.sign(W) * margin / np.sqrt(d)
    b = rng.normal(size=kp)
    return X, y, np.arange(K, dtype=np.float64), W, b


def _eval(ctx, Xd, yd, classes, W, b, **opts):
    """(loss, dW, db) and the path that ran"""
    with _options(ctx, **opts):
        loss, gW, gb, nt = ctx.logreg_eval(Xd, yd, classes, W, b)
        path = ctx.stats()["last_path"]
    assert nt == Xd.shape[0]
    return (loss, gW, gb), path


def _within(res, ref, bd, scale, what):
    loss, gW, gb = res
    assert abs(loss - ref[0]) <= scale * bd["loss"], (what, "loss", loss, ref[0], bd["loss"])
    eW, eb = np.abs(gW - ref[1]), np.abs(gb - ref[2])
    assert np.all(eW <= scale * bd["dW"]), (what, "dW", float(eW.max()), float((eW / bd["dW"]).max()))
    assert np.all(eb <= scale * bd["db"]), (what, "db", float(eb.max()), float(bd["db"].max()))


def _same_bits(a, c):
    return a[0] == c[0] and np.array_equal(a[1], c[1]) and np.array_equal(a[2], c[2])


# ---------------------------------------------------------------------------------------------------------------------
# a. the fused pass with many tiles per CTA
# ---------------------------------------------------------------------------------------------------------------------
# (d, K'): every instantiation at the largest d it takes; ragged K' at tiny d; each side of every tile-height change
LIMIT_SHAPES = [(1024, 1), (1024, 2), (1024, 4), (512, 8), (256, 16), (128, 17)]
SMALL_SHAPES = [(d, kp) for d in (1, 3) for kp in (3, 5, 7, 9, 17)]
TILE_EDGES = [(128, 16), (129, 16), (128, 6), (129, 6), (256, 8), (257, 8), (256, 2), (257, 2), (512, 3), (513, 3),
              (512, 1), (513, 1)]
STEADY = ([(d, kp, {}) for d, kp in LIMIT_SHAPES + SMALL_SHAPES + TILE_EDGES]
          # features offset by 1e3, one per tile height
          + [(d, kp, {"offset": 1e3, "wscale": 1e-3}) for d, kp in ((64, 1), (200, 4), (400, 8), (1000, 2))]
          # margins of +-1e3 at KB = 8
          + [(64, 6, {"margin": 1e3})])


@pytest.mark.parametrize("d,kp,opts", STEADY,
                         ids=[f"d{d}-k{kp}" + "".join(f"-{k}" for k in o) for d, kp, o in STEADY])
def test_fused_pass_in_steady_state(ctx, d, kp, opts):
    """Per tile, the next one streams into the other half of a double buffer and the loss and intercept sums carry
    across tiles in shared memory: at N rows with 1, 3 or 7 CTAs, and at the default grid with at least 5 tiles per
    CTA, the auto path is the fused pass, within the fp64 bound of the oracle, within twice it of the generic pass, and
    bitwise reproducible at each grid."""
    assert fused_covers(d, kp)
    tr = tile_rows(d)
    sm = _sm_count()
    for n, limits in ((N, GRID_LIMITS), (MIN_TILES_PER_CTA * tr * MAX_CTAS_PER_SM * sm + 37, (0,))):
        assert n % tr != 0   # a ragged last tile
        for gl in limits:    # the schedule the grid gives: many tiles per CTA
            span_rows, grid = fused_spans(n, d, gl if gl else MAX_CTAS_PER_SM * sm)
            assert span_rows // tr >= MIN_TILES_PER_CTA and grid <= (gl or MAX_CTAS_PER_SM * sm), (n, gl, span_rows)
        X, y, classes, W, b = _case(n, d, kp, seed=7 * d + kp, **opts)
        ref = lo.loss_grad(X, np.searchsorted(classes, y.astype(np.float64)), W, b)
        bd = lo.eval_bound(X, W, b)
        Xd, yd = torch.from_numpy(X).cuda(), torch.from_numpy(y).cuda()
        gen, path = _eval(ctx, Xd, yd, classes, W, b, kernel_path=1)
        assert path == 1
        _within(gen, ref, bd, 1.0, ("generic", n))
        for gl in limits:
            a, path = _eval(ctx, Xd, yd, classes, W, b, grid_limit=gl)
            assert path == 2, f"auto did not take the fused pass at d = {d}, K' = {kp}"
            c, _ = _eval(ctx, Xd, yd, classes, W, b, grid_limit=gl)
            _within(a, ref, bd, 1.0, ("fused", n, gl))
            _within(a, gen, bd, 2.0, ("fused - generic", n, gl))
            assert _same_bits(a, c), f"two fused evaluations differ at n = {n}, grid_limit = {gl}"
            if "margin" in opts:
                assert np.isfinite(a[0]) and np.all(np.isfinite(a[1])) and np.all(np.isfinite(a[2]))
        del Xd, yd


def test_grid_limit_zero_is_the_default_grid(ctx):
    X, y, classes, W, b = _case(N, 130, 10, seed=5)
    Xd, yd = torch.from_numpy(X).cuda(), torch.from_numpy(y).cuda()
    a, _ = _eval(ctx, Xd, yd, classes, W, b)
    c, _ = _eval(ctx, Xd, yd, classes, W, b, grid_limit=100000)   # larger than the default grid: no cap
    assert _same_bits(a, c)


# ---------------------------------------------------------------------------------------------------------------------
# b. where the fused pass stops
# ---------------------------------------------------------------------------------------------------------------------
def _smem_edge_at_d1():
    kp = 1
    while fused_covers(1, kp + 1):
        kp += 1
    return kp


def test_fused_coverage_limits(ctx):
    """Just inside each limit auto takes the fused pass; just outside it takes the generic one and a forced fused pass
    fails.  At d = 1 shared memory is the limit: [K'][d] weights and [tr][K'] margins, residuals and intercept sums."""
    last = _smem_edge_at_d1()
    assert fused_pick(1, last + 1) is not None   # the accumulators would still cover it
    pairs = [((256, 16), (257, 16)), ((128, 17), (129, 17)), ((512, 8), (513, 8)), ((1, last), (1, last + 1))]
    for inside, outside in pairs:
        assert fused_covers(*inside) and not fused_covers(*outside), (inside, outside)
        for (d, kp), fused in ((inside, True), (outside, False)):
            X, y, classes, W, b = _case(777, d, kp, seed=d + kp)
            Xd, yd = torch.from_numpy(X).cuda(), torch.from_numpy(y).cuda()
            res, path = _eval(ctx, Xd, yd, classes, W, b)
            assert path == (2 if fused else 1), (d, kp, path)
            _within(res, lo.loss_grad(X, y.astype(np.int64), W, b), lo.eval_bound(X, W, b), 1.0, (d, kp))
            if not fused:
                with pytest.raises(_native.B2KError, match="does not cover"):
                    _eval(ctx, Xd, yd, classes, W, b, kernel_path=2)


# ---------------------------------------------------------------------------------------------------------------------
# c. the generic pass over several chunks
# ---------------------------------------------------------------------------------------------------------------------
def _generic_cases():
    c40, c1 = generic_chunk(1 << 30, 40), generic_chunk(1 << 30, 1)
    # (d, K', n): 3 chunks with a ragged last one at d % 4 != 0 (scalar loads) and d % 4 == 0; 3 chunks at K' = 40;
    # 2 chunks at K' = 1
    return [(5, 1024, N), (8, 1024, N), (4, 40, 2 * c40 + c40 // 5 + 11), (2, 1, c1 + 4097)]


@pytest.mark.parametrize("d,kp,n", _generic_cases())
def test_generic_pass_over_several_chunks(ctx, d, kp, n):
    chunk = generic_chunk(n, kp)
    assert _cdiv(n, chunk) >= 2 and n % chunk != 0, (n, chunk)
    X, y, classes, W, b = _case(n, d, kp, seed=n % 1000 + kp)
    ref = lo.loss_grad(X, y.astype(np.int64), W, b)
    bd = lo.eval_bound(X, W, b)
    Xd, yd = torch.from_numpy(X).cuda(), torch.from_numpy(y).cuda()
    a, path = _eval(ctx, Xd, yd, classes, W, b, kernel_path=1)
    c, _ = _eval(ctx, Xd, yd, classes, W, b, kernel_path=1)
    assert path == 1
    _within(a, ref, bd, 1.0, ("generic", n, chunk))
    assert _same_bits(a, c)


# ---------------------------------------------------------------------------------------------------------------------
# d. an X that is not 16-byte aligned
# ---------------------------------------------------------------------------------------------------------------------
def _unaligned(X):
    n, d = X.shape
    buf = torch.zeros(n * d + 1, dtype=torch.float32, device="cuda")
    buf[1:] = torch.from_numpy(X.reshape(-1)).cuda()
    Xu = buf[1:].view(n, d)
    assert Xu.data_ptr() % 16 == 4
    return Xu


@pytest.mark.parametrize("d,kp", [(64, 3), (128, 1), (1024, 9)])
def test_unaligned_rows_give_the_same_bits(ctx, d, kp):
    """The float4 and scalar loads read the same features in the same order: an X one float into its buffer gives
    the bits of an aligned copy on both evaluation paths and in the transform."""
    X, y, classes, W, b = _case(N, d, kp, seed=d + 3 * kp)
    Xa, Xu, yd = torch.from_numpy(X).cuda(), _unaligned(X), torch.from_numpy(y).cuda()
    for path in ((1, 2) if fused_covers(d, kp) else (1,)):
        a, _ = _eval(ctx, Xa, yd, classes, W, b, kernel_path=path)
        u, _ = _eval(ctx, Xu, yd, classes, W, b, kernel_path=path)
        assert _same_bits(a, u), f"path {path}: an unaligned X changes the evaluation"
    cv = np.arange(2 if kp == 1 else kp, dtype=np.float64)
    for ta, tu in zip(ctx.logreg_predict(Xa, W, b, cv), ctx.logreg_predict(Xu, W, b, cv)):
        assert torch.equal(ta, tu), "an unaligned X changes the transform"


# ---------------------------------------------------------------------------------------------------------------------
# e. rows whose label is none of the classes
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("classes", [[0.0, 2.0, 3.0], [1.0, 4.0]], ids=["multinomial", "binomial"])
def test_rows_of_no_class(ctx, classes):
    """b2k_logreg_eval counts a row whose label is not one of `classes` (another class value, >= 1024, negative or
    fractional) as no class: a zero one-hot, for binomial a negative row."""
    classes = np.array(classes)
    kp = 1 if len(classes) == 2 else len(classes)
    d = 24
    rng = np.random.default_rng(len(classes))
    X = rng.standard_normal(size=(N, d), dtype=np.float32)
    y = rng.choice(np.array([0, 1, 2, 3, 4, 5, 1024, 5000, 1e9, -1, 2.5], dtype=np.float32), size=N)
    W, b = rng.normal(size=(kp, d)) / np.sqrt(d), rng.normal(size=kp)
    idx = {float(c): i for i, c in enumerate(classes)}
    yi = np.array([idx.get(float(v), -1) for v in y])
    assert np.any(yi < 0) and all(np.any(yi == i) for i in range(len(classes)))
    ref = lo.loss_grad(X, yi, W, b)
    bd = lo.eval_bound(X, W, b)
    Xd, yd = torch.from_numpy(X).cuda(), torch.from_numpy(y).cuda()
    for opts in ({"kernel_path": 1}, {"kernel_path": 2}, {"kernel_path": 2, "grid_limit": 3}):
        res, _ = _eval(ctx, Xd, yd, classes, W, b, **opts)
        _within(res, ref, bd, 1.0, opts)


# ---------------------------------------------------------------------------------------------------------------------
# f. the label pass at its span cap
# ---------------------------------------------------------------------------------------------------------------------
def _labels(ctx, y):
    return ctx.logreg_labels(torch.from_numpy(y).cuda())


def _capped_n():
    n = 3 * 4 * _sm_count() * LABEL_SPAN_ROWS + 77
    spans, span_rows = label_spans(n)
    assert spans == 4 * _sm_count() and n - (spans - 1) * span_rows < span_rows   # capped, a short last span
    return n, spans, span_rows


def test_labels_at_the_span_cap_count_every_class_exactly(ctx):
    n, _, _ = _capped_n()
    rng = np.random.default_rng(17)
    y = rng.integers(0, MAX_CLASSES, size=n).astype(np.float32)
    rows = rng.permutation(n)
    y[rows[:MAX_CLASSES]] = np.arange(MAX_CLASSES)
    y[rows[MAX_CLASSES:MAX_CLASSES + 1000]] = -0.0   # -0.0 is class 0
    classes, counts, nt = _labels(ctx, y)
    cls_ref, cnt_ref = np.unique(y.astype(np.float64), return_counts=True)
    assert nt == n and np.array_equal(classes, np.arange(MAX_CLASSES, dtype=np.float64))
    assert np.array_equal(classes, cls_ref) and np.array_equal(counts, cnt_ref)


def test_labels_count_past_2_to_the_24(ctx):
    """fp32 would stop counting at 2^24: the per-span counts are integers, folded in fp64"""
    n = 20_000_000
    rng = np.random.default_rng(19)
    y = np.zeros(n, dtype=np.float32)
    some = rng.permutation(n)[:n // 100]
    y[some] = rng.integers(1, 7, size=some.size)
    classes, counts, nt = _labels(ctx, y)
    cnt_ref = np.bincount(y.astype(np.int64))
    assert counts[0] > 2 ** 24 and nt == n
    assert np.array_equal(classes, np.flatnonzero(cnt_ref)) and np.array_equal(counts, cnt_ref[cnt_ref > 0])


@pytest.mark.parametrize("bad,msg", [
    (-1.0, r"Labels MUST be in \[0, 2147483647\), but got -1\.0"),
    (0.5, r"Labels MUST be Integers, but got 0\.5"),
    (1024.0, r"supports label values below 1024 \(at most 1024 classes\), got 1024\.0"),
    (float("nan"), "the label holds a NaN or an infinity"),
    (float("inf"), "the label holds a NaN or an infinity"),
    (float("-inf"), "the label holds a NaN or an infinity")])
def test_labels_report_a_bad_value_in_any_span(ctx, bad, msg):
    n, spans, span_rows = _capped_n()
    y = (np.arange(n) % 1023).astype(np.float32)
    for row in (n - 1, spans // 2 * span_rows):   # the last row of the last span, the first row of a middle one
        yb = y.copy()
        yb[row] = bad
        with pytest.raises(_native.B2KError, match=msg):
            _labels(ctx, yb)
    yb = y.copy()
    yb[n - 1] = 1023.0   # the largest class value is valid
    classes, counts, _ = _labels(ctx, yb)
    assert classes[-1] == 1023.0 and counts[-1] == 1 and len(classes) == 1024


# ---------------------------------------------------------------------------------------------------------------------
# g. the transform kernel over several sweeps of its grid
# ---------------------------------------------------------------------------------------------------------------------
def _predict(ctx, X, W, b, cv):
    raw, prob, pred = ctx.logreg_predict(torch.from_numpy(X).cuda(), W, b, cv)
    return raw.cpu().numpy(), prob.cpu().numpy(), pred.cpu().numpy()


def _check_predict(X, W, b, cv, raw, prob, pred):
    d, kp = X.shape[1], W.shape[0]
    o = lo.predict(X, W, b, cv)
    A = np.abs(X.astype(np.float64)) @ np.abs(W).T + np.abs(b)   # [n, kp] |margin| scale
    e_m = (d + 4) * U * A + 16 * U                                 # per margin
    em = e_m.max(axis=1)                                           # per row, any class
    e_r = 2 * kp * em + 16 * U                                     # residual (probability) bound of eval_bound
    if kp == 1:
        e_m = np.concatenate([e_m, e_m], axis=1)
    err = np.abs(raw - o["raw"])
    assert np.all(err <= e_m), ("raw", float((err / e_m).max()))
    err = np.abs(prob - o["prob"])
    assert np.all(err <= e_r[:, None]), ("probability", float((err / e_r[:, None]).max()))
    s = np.abs(prob.sum(axis=1) - 1.0)
    assert np.all(s <= max(kp, 2) * 4 * U), ("probability sum", float(s.max()))
    if kp == 1:
        gap = np.abs(o["raw"][:, 1])
    else:
        top2 = np.partition(o["raw"], kp - 2, axis=1)[:, kp - 2:]
        gap = top2[:, 1] - top2[:, 0]
    clear = gap > 2 * em
    assert clear.mean() > 0.9
    assert np.array_equal(pred[clear], o["pred"][clear]), "prediction"


PREDICT_D = [1, 3, 4, 64, 65, 127, 128, 1024]


@pytest.mark.parametrize("d", PREDICT_D)
def test_transform_over_several_sweeps(ctx, d):
    """raw within the margin bound, probabilities within the residual bound and summing to 1, and the oracle's
    prediction wherever the top two margins are clearly apart, over 3 sweeps of the grid and a ragged fourth, for
    binomial and K' = 3, 8, 9 and 17 (and 1024 where a sweep is short): a second 8-class pass of the k0 loop, L = 1 to
    32 lanes per row, scalar and float4 loads, class values that are not 0, 1, ..."""
    sweep = predict_sweep(d)
    n = 3 * sweep + 37
    rng = np.random.default_rng(d)
    X = rng.standard_normal(size=(n, d), dtype=np.float32)
    for kp in [1, 3, 8, 9, 17] + ([1024] if row_lanes(d) == 32 else []):
        nout = 2 if kp == 1 else kp
        W, b = rng.normal(size=(kp, d)) * 2 / np.sqrt(d), rng.normal(size=kp)
        cv = np.sort(rng.choice(4 * nout, size=nout, replace=False)).astype(np.float64)
        raw, prob, pred = _predict(ctx, X, W, b, cv)
        assert raw.shape == (n, nout) and pred.shape == (n,)
        _check_predict(X, W, b, cv, raw, prob, pred)


def test_transform_edges(ctx):
    rng = np.random.default_rng(23)
    n, d = 1000, 12
    X = rng.standard_normal(size=(n, d), dtype=np.float32)
    # an exact tie across the two 8-class passes predicts the first class, as MLlib's argmax does
    kp = 17
    W, b = rng.normal(size=(kp, d)) / np.sqrt(d), rng.normal(size=kp)
    W[11], b[2], b[11] = W[2], 50.0, 50.0
    cv = np.arange(kp, dtype=np.float64) * 2
    raw, prob, pred = _predict(ctx, X, W, b, cv)
    assert np.array_equal(raw[:, 2], raw[:, 11]) and np.all(pred == cv[2])
    assert np.array_equal(prob[:, 2], prob[:, 11])
    # m = 0 (binomial): class_values[0], [0.5, 0.5]; all margins equal (multinomial): the first class, 1/K' each
    raw, prob, pred = _predict(ctx, X, np.zeros((1, d)), np.zeros(1), np.array([3.0, 7.0]))
    assert np.all(raw == 0.0) and np.all(prob == 0.5) and np.all(pred == 3.0)
    raw, prob, pred = _predict(ctx, X, np.zeros((4, d)), np.zeros(4), np.array([3.0, 7.0, 9.0, 11.0]))
    assert np.all(raw == 0.0) and np.all(prob == 0.25) and np.all(pred == 3.0)
    # margins of +-1e3 (+-1 features, exact margins, no ties): finite, exactly 0 or 1 where fp64 says so
    Xs = rng.choice(np.array([-1.0, 1.0], dtype=np.float32), size=(n, 4))
    for kp in (1, 3):
        W = rng.choice([-250.0, 250.0], size=(kp, 4))
        b = np.arange(kp) * 0.25 + 0.125
        cv = np.arange(2 if kp == 1 else kp, dtype=np.float64)
        raw, prob, pred = _predict(ctx, Xs, W, b, cv)
        o = lo.predict(Xs, W, b, cv)
        assert np.all(np.isfinite(prob)) and np.abs(raw).max() >= 1e3
        hard = (o["prob"] == 0.0) | (o["prob"] == 1.0)
        assert hard.any() and np.array_equal(prob[hard], o["prob"][hard])
        _check_predict(Xs, W, b, cv, raw, prob, pred)
        assert np.array_equal(pred, o["pred"])   # margins exact: no row is near a tie it could resolve otherwise
    # the one-label model: b = +-inf, W = 0
    for inf, p, c in ((np.inf, [0.0, 1.0], 1.0), (-np.inf, [1.0, 0.0], 0.0)):
        raw, prob, pred = _predict(ctx, X, np.zeros((1, d)), np.array([inf]), np.array([0.0, 1.0]))
        assert np.all(raw == [-inf, inf]) and np.all(prob == p) and np.all(pred == c)


@pytest.mark.parametrize("d", [7, 40])
def test_linreg_predict_over_several_sweeps(ctx, d):
    """k_linreg_predict's grid-stride loop past its first sweep, against the bound of test_gpu_linreg.py"""
    n = 3 * predict_sweep(d) + 37
    rng = np.random.default_rng(d)
    X = rng.standard_normal(size=(n, d), dtype=np.float32) + np.float32(2.0)
    w, icpt = rng.normal(size=d), 0.75
    pred = ctx.linreg_predict(torch.from_numpy(X).cuda(), w, icpt).cpu().numpy()
    terms = X.astype(np.float64) * w
    ref = icpt + terms.sum(1)
    bound = d * 2.0 ** -52 * (np.abs(terms).sum(1) + abs(icpt))
    assert pred.shape == (n,) and np.all(np.abs(pred - ref) <= bound)


# ---------------------------------------------------------------------------------------------------------------------
# h. one fit in steady state
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("path", [2, 1])
def test_fit_at_a_capped_grid_reaches_the_optimum(ctx, path):
    """K = 6 (KB = 8), d = 40, n = 60000 through b2k_logreg_fit with 5 CTAs: every evaluation of the optimisation
    runs many tiles per CTA"""
    n, d, K = 60000, 40, 6
    assert fused_covers(d, K) and fused_spans(n, d, 5)[0] // tile_rows(d) >= 100
    rng = np.random.default_rng(29)
    X = (rng.normal(size=(n, d)) * (1 + np.arange(d) % 3)).astype(np.float32)
    Wt = rng.normal(size=(K, d)) / np.sqrt(d)
    y = (X.astype(np.float64) @ Wt.T + rng.gumbel(size=(n, K))).argmax(1).astype(np.float32)
    Xd, yd = torch.from_numpy(X).cuda(), torch.from_numpy(y).cuda()
    classes, counts, _ = ctx.logreg_labels(yd)
    assert np.array_equal(classes, np.arange(K))
    s = {"reg": 0.01, "l1_ratio": 0.0, "tol": 1e-12, "max_iter": 1000, "fit_intercept": True,
         "standardization": True, "family": "auto"}
    with _options(ctx, kernel_path=path, grid_limit=5):
        (W, b, _), = ctx.logreg_fit(Xd, yd, classes, counts, [s])
        assert ctx.stats()["last_path"] == path
    P = lo.Problem(X, y, 0.01, 0.0, True, True)
    theta = np.concatenate([(W * P.sig).ravel(), b])   # centred multinomial intercepts: the same loss
    x, _, _, _ = _native.logreg_minimize(P.smooth, P.start(), None, 1000, 1e-12)
    assert P.residual(theta) <= max(1e-8, 1.5 * P.residual(x)), (P.residual(theta), P.residual(x))
