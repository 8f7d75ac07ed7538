"""b2k_mlp_eval / b2k_mlp_fit / b2k_mlp_predict on the device against the fp64 oracle (tests/mlp_oracle.py): both paths
over the widths, class counts and depths at their edges and past a row chunk, saturated sigmoids, a capped grid in
steady state, bitwise repeats and grid invariance, fits of both solvers against an oracle-driven run of the same
minimiser, prediction, and every error path."""
import numpy as np
import pytest

import mlp_oracle as mo

pytestmark = pytest.mark.gpu

UNIT = 4096
CHUNK_BYTES = 32 << 20


@pytest.fixture(scope="module")
def ctx():
    from spark_rapids_ml_b200._native import Context

    c = Context(0)
    yield c
    c.close()


@pytest.fixture(autouse=True)
def _reset(ctx):
    yield
    ctx.set_option("kernel_path", 0)
    ctx.set_option("grid_limit", 0)
    ctx.set_option("time_kernels", 0)


def _dev(a, dtype=np.float32):
    import torch

    return torch.from_numpy(np.ascontiguousarray(a, dtype=dtype)).cuda()


def chunk_rows(layers, n, es):
    """The rows per chunk the header states."""
    per_row = 8 + es * sum((w + 3) // 4 * 4 for w in layers[1:])
    R = max(1, CHUNK_BYTES // per_row // UNIT) * UNIT
    return min(R, max(1, -(-n // UNIT)) * UNIT)


def _data(n, layers, seed, shift=0.0, scale=1.0):
    rng = np.random.default_rng(seed)
    X = (rng.normal(size=(n, layers[0])) * scale + shift).astype(np.float32)
    y = rng.integers(0, layers[-1], size=n).astype(np.float32)
    w = rng.normal(size=mo.n_weights(layers)) * 0.5
    return X, y, w


def _check_eval(ctx, layers, X, y, w, path):
    ctx.set_option("kernel_path", path)
    F, g, nt = ctx.mlp_eval(_dev(X), _dev(y), layers, w)
    assert nt == len(X)
    Fo, go = mo.eval_fg(layers, w, X.astype(np.float64), y)
    bF, bg = mo.eval_bound(layers, w, X.astype(np.float64), y)
    assert abs(F - Fo) <= bF, (F, Fo, bF)
    bad = np.abs(g - go) > bg + 1e-300
    assert not bad.any(), (np.flatnonzero(bad)[:5], g[bad][:5], go[bad][:5], bg[bad][:5])
    return ctx.stats()["last_path"]


EVAL_CASES = [
    ([1, 2], 1), ([3, 10], 50), ([3, 1, 2], 7), ([64, 63, 10], 300), ([128, 64, 65], 257), ([64, 65, 64, 2], 1000),
    ([128, 129, 63, 1, 10], 513), ([784, 129, 10], 200), ([4, 64, 64, 64, 65], 100), ([128, 64, 32, 10], 3000),
]


@pytest.mark.parametrize("layers,n", EVAL_CASES)
@pytest.mark.parametrize("path", [1, 0])
def test_eval_matches_oracle(ctx, layers, n, path):
    X, y, w = _data(n, layers, seed=n + len(layers))
    got = _check_eval(ctx, layers, X, y, w, path)
    assert got == (2 if path == 0 and layers[0] % 4 == 0 else 1)


@pytest.mark.parametrize("path", [1, 2])
def test_eval_past_a_chunk(ctx, path):
    layers = [64, 65, 10]
    R = chunk_rows(layers, 1 << 30, 4 if path == 2 else 8)
    n = R + 1234
    X, y, w = _data(n, layers, seed=3)
    _check_eval(ctx, layers, X, y, w, path)


@pytest.mark.parametrize("shift,scale", [(20.0, 1.0), (0.0, 30.0)])
@pytest.mark.parametrize("path", [1, 2])
def test_eval_saturated(ctx, shift, scale, path):
    layers = [16, 63, 65, 3]
    X, y, w = _data(700, layers, seed=5, shift=shift, scale=scale)
    _check_eval(ctx, layers, X, y, w, path)


def test_eval_steady_state_and_grid_invariance(ctx):
    layers = [64, 64, 10]
    R = chunk_rows(layers, 1 << 30, 4)
    n = 2 * R + 999
    X, y, w = _data(n, layers, seed=9)
    Xd, yd = _dev(X), _dev(y)
    outs = []
    for gl in (0, 3, 7):
        ctx.set_option("kernel_path", 2)
        ctx.set_option("grid_limit", gl)
        outs.append(ctx.mlp_eval(Xd, yd, layers, w))
    again = ctx.mlp_eval(Xd, yd, layers, w)
    for F, g, _ in outs[1:] + [again]:
        assert F == outs[0][0]
        assert np.array_equal(g, outs[0][1])
    Fo, go = mo.eval_fg(layers, w, X.astype(np.float64), y)
    bF, bg = mo.eval_bound(layers, w, X.astype(np.float64), y)
    assert abs(outs[0][0] - Fo) <= bF
    assert (np.abs(outs[0][1] - go) <= bg).all()


def test_generic_repeat_bitwise(ctx):
    layers = [3, 65, 2]
    X, y, w = _data(5000, layers, seed=11)
    Xd, yd = _dev(X), _dev(y)
    ctx.set_option("grid_limit", 5)
    a = ctx.mlp_eval(Xd, yd, layers, w)
    ctx.set_option("grid_limit", 0)
    b = ctx.mlp_eval(Xd, yd, layers, w)
    assert a[0] == b[0] and np.array_equal(a[1], b[1])


@pytest.mark.parametrize("solver", ["l-bfgs", "gd"])
@pytest.mark.parametrize("path", [1, 2])
def test_fit_matches_oracle_minimiser(ctx, solver, path):
    from spark_rapids_ml_b200._native import logreg_minimize

    layers = [8, 5, 3]
    rng = np.random.default_rng(21)
    X = rng.normal(size=(600, 8)).astype(np.float32)
    y = (np.argmax(X[:, :3], axis=1)).astype(np.float32)
    ctx.set_option("kernel_path", path)
    it = 6
    res = ctx.mlp_fit(_dev(X), _dev(y), layers, solver=solver, max_iter=it, tol=0.0, step_size=0.5, seed=4)
    w0 = mo.init_weights(layers, 4)
    fun = lambda w: mo.eval_fg(layers, w, X.astype(np.float64), y)   # noqa: E731
    if solver == "l-bfgs":
        wo, n_it, _, fo = logreg_minimize(fun, w0, max_iter=it, tol=0.0)
        assert res["n_iter"] == n_it + 1
        assert abs(res["objective_history"][-1] - fo) <= 1e-4 * abs(fo)
        f0 = fun(w0)[0]
        assert abs(res["objective_history"][0] - f0) <= 1e-5 * abs(f0)
    else:
        wo, hist = mo.gd(fun, w0, it, 0.0, 0.5)
        assert res["n_iter"] == len(hist) == it
        np.testing.assert_allclose(res["objective_history"], hist, rtol=1e-5)
    np.testing.assert_allclose(res["weights"], wo, rtol=1e-3, atol=1e-4)


def test_fit_initial_weights_and_history_descends(ctx):
    layers = [8, 6, 3]
    rng = np.random.default_rng(2)
    X = rng.normal(size=(2000, 8)).astype(np.float32)
    y = (np.argmax(X[:, :3] + 0.1 * rng.normal(size=(2000, 3)), axis=1)).astype(np.float32)
    w0 = rng.normal(size=mo.n_weights(layers)) * 0.1
    res = ctx.mlp_fit(_dev(X), _dev(y), layers, max_iter=30, initial_weights=w0)
    h = res["objective_history"]
    assert abs(h[0] - mo.eval_fg(layers, w0, X.astype(np.float64), y)[0]) <= 1e-5 * h[0]
    assert (np.diff(h) <= 1e-12).all()
    assert h[-1] < 0.5 * h[0]


@pytest.mark.parametrize("path", [1, 2])
def test_predict_matches_oracle(ctx, path):
    layers = [128, 64, 32, 10]
    X, _, w = _data(9000, layers, seed=13)
    ctx.set_option("kernel_path", path)
    raw, prob, pred = ctx.mlp_predict(_dev(X), layers, w)
    z, p, pr = mo.predict(layers, w, X.astype(np.float64))
    _, bz = mo.z_bound(layers, w, X.astype(np.float64))
    raw, prob, pred = raw.cpu().numpy(), prob.cpu().numpy(), pred.cpu().numpy()
    assert (np.abs(raw - z) <= bz).all()
    np.testing.assert_allclose(prob, p, atol=2 * bz.max() + 1e-12)
    top2 = np.sort(z, axis=1)[:, -2:]
    clear = top2[:, 1] - top2[:, 0] > 2 * bz.max(axis=1)
    assert np.array_equal(pred[clear], pr[clear])
    assert clear.mean() > 0.99


def test_errors(ctx):
    from spark_rapids_ml_b200._native import B2KError

    layers = [4, 3, 2]
    X, y, w = _data(50, layers, seed=1)
    Xd, yd = _dev(X), _dev(y)
    bad_y = y.copy()
    bad_y[3] = 2.0
    with pytest.raises(B2KError, match="labels must be in \\[0, 2\\)"):
        ctx.mlp_eval(Xd, _dev(bad_y), layers, w)
    bad_y[3] = 0.5
    with pytest.raises(B2KError, match="Labels MUST be Integers"):
        ctx.mlp_fit(Xd, _dev(bad_y), layers, max_iter=2)
    bad_y[3] = -1.0
    with pytest.raises(B2KError, match="Labels MUST be in"):
        ctx.mlp_eval(Xd, _dev(bad_y), layers, w)
    Xn = X.copy()
    Xn[7, 2] = np.nan
    for path in (1, 2):
        ctx.set_option("kernel_path", path)
        with pytest.raises(B2KError, match="NaN or an infinity"):
            ctx.mlp_eval(_dev(Xn), yd, layers, w)
    ctx.set_option("kernel_path", 0)
    wn = w.copy()
    wn[0] = np.inf
    with pytest.raises(B2KError, match="weight is not finite"):
        ctx.mlp_eval(Xd, yd, layers, wn)
    with pytest.raises(B2KError, match="weight is not finite"):
        ctx.mlp_predict(Xd, layers, wn)
    with pytest.raises(B2KError, match="at least 2 entries"):
        ctx.mlp_eval(Xd, yd, [4], np.zeros(0))
    with pytest.raises(B2KError, match="must be >= 1"):
        ctx.mlp_eval(Xd, yd, [4, 0, 2], np.zeros(mo.n_weights([4, 0, 2])))
    with pytest.raises(B2KError, match="widths <= 1024") as e:
        ctx.mlp_eval(Xd, yd, [4, 1025, 2], np.zeros(mo.n_weights([4, 1025, 2])))
    assert e.value.code == 4
    with pytest.raises(ValueError, match="must equal the feature count"):
        ctx.mlp_eval(Xd, yd, [5, 2], np.zeros(12))
    with pytest.raises(B2KError, match="maxIter given invalid value -1"):
        ctx.mlp_fit(Xd, yd, layers, max_iter=-1)
    with pytest.raises(B2KError, match="tol must be >= 0"):
        ctx.mlp_fit(Xd, yd, layers, tol=-1.0)
    with pytest.raises(B2KError, match="stepSize must be > 0"):
        ctx.mlp_fit(Xd, yd, layers, solver="gd", step_size=0.0)
    X3, y3, w3 = _data(20, [3, 2], seed=2)
    ctx.set_option("kernel_path", 2)
    with pytest.raises(B2KError, match="kernel_path=2") as e:
        ctx.mlp_eval(_dev(X3), _dev(y3), [3, 2], w3)
    assert e.value.code == 4
    with pytest.raises(B2KError, match="kernel_path=2"):
        ctx.mlp_predict(_dev(X3), [3, 2], w3)
    ctx.set_option("kernel_path", 0)
    with pytest.raises(B2KError, match="empty partition"):
        ctx.mlp_eval(_dev(np.zeros((0, 4))), _dev(np.zeros(0)), layers, w)


def test_timing_stats(ctx):
    layers = [16, 8, 3]
    X, y, w = _data(3000, layers, seed=6)
    ctx.set_option("time_kernels", 1)
    ctx.mlp_fit(_dev(X), _dev(y), layers, max_iter=3)
    st = ctx.stats()
    assert st["last_fused_ms"] > 0 and st["last_loop_ms"] >= st["last_fused_ms"]
    assert st["last_path"] == 2
