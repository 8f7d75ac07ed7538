"""DBSCAN on one H100: b2k_dbscan_fit's labels, core flags and cluster count must equal the fp64 oracle of
tests/dbscan_oracle.py bit for bit, on both passes, at every DP width, far from the origin, on pairs exactly at and one
ulp around eps, on chains that span many blocks and splits, under a persistent schedule squeezed onto few CTAs, and at
ragged row counts.  Errors must be the documented ones."""
import numpy as np
import pyarrow as pa
import pytest

import dbscan_oracle as do

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from spark_rapids_ml_b200 import _native  # noqa: E402


@pytest.fixture(scope="module")
def ctx():
    with _native.Context(0) as c:
        yield c


def _fit(ctx, X, eps, ms, metric="euclidean", path=0, grid=0, recheck=0):
    """(labels, core, n_clusters, stats) of one call on X (numpy)."""
    ctx.set_option("kernel_path", path)
    ctx.set_option("grid_limit", grid)
    ctx.set_option("collect_recheck", recheck)
    try:
        lab, core, ncl = ctx.dbscan_fit(torch.from_numpy(np.ascontiguousarray(X)).cuda(), eps, ms, metric)
        return lab.cpu().numpy(), core.cpu().numpy(), ncl, ctx.stats()
    finally:
        ctx.set_option("kernel_path", 0)
        ctx.set_option("grid_limit", 0)
        ctx.set_option("collect_recheck", 0)


def _wg_ok(d):
    return d % 4 == 0 and 4 <= d <= 128


def _paths(d):
    return [2, 1] if _wg_ok(d) else [1]


def _check(ctx, X, eps, ms, metric="euclidean", paths=None, grid=0):
    ref = do.dbscan(X, eps, ms, metric)
    for path in paths or _paths(X.shape[1]):
        lab, core, ncl, st = _fit(ctx, X, eps, ms, metric, path, grid)
        assert st["last_path"] == path
        assert ncl == ref[2], (path, ncl, ref[2])
        np.testing.assert_array_equal(core, ref[1], err_msg=f"core flags, path {path}")
        np.testing.assert_array_equal(lab, ref[0], err_msg=f"labels, path {path}")
    return ref


def blobs(n, d, k, seed, spread=10.0, std=1.0, offset=0.0):
    rng = np.random.default_rng(seed)
    C = rng.uniform(-spread, spread, size=(k, d))
    X = C[rng.integers(0, k, size=n)] + std * rng.normal(size=(n, d)) + offset
    return X.astype(np.float32)


# ---- shapes and data ----
def test_reference_shape_blobs(ctx):
    """The reference's test_dbscan shape: 1000 x 20 blobs, eps = 5, min_samples = 5."""
    X = blobs(1000, 20, 5, seed=0, spread=10.0, std=1.0)
    ref = _check(ctx, X, 5.0, 5)
    assert ref[2] >= 2 and (ref[0] == -1).sum() < len(X)


@pytest.mark.parametrize("d", [4, 128, 200])
def test_widths(ctx, d):
    X = blobs(1200, d, 6, seed=d, spread=3.0, std=1.0)
    eps = float(0.85 * np.sqrt(2 * d))
    ref = _check(ctx, X, eps, 4)
    assert ref[2] >= 1


@pytest.mark.parametrize("d", [8, 40, 96])
def test_far_from_origin(ctx, d):
    """+1e3 on every feature: the shifted frame keeps the screen's error at the data's spread."""
    X = blobs(1500, d, 5, seed=10 + d, spread=2.0, std=0.5, offset=1e3)
    _check(ctx, X, float(0.85 * 0.5 * np.sqrt(2 * d)), 5)


def test_integer_pairs_exactly_at_eps(ctx):
    """Integer rows, eps = 3: pairs at distance exactly 3 count (<=), pairs at sqrt(10) do not."""
    rng = np.random.default_rng(5)
    base = rng.integers(-1000, 1000, size=(300, 8)) * 10
    X = np.concatenate([base, base + np.array([3, 0, 0, 0, 0, 0, 0, 0]),
                        base + np.array([0, 3, 1, 0, 0, 0, 0, 0])]).astype(np.float32)
    ref = _check(ctx, X, 3.0, 2)
    assert ref[1][:600].all() and not ref[1][600:].any()


def _ulp_pairs(n_pairs, d, seed, eps=0.75):
    """Pairs along feature 0 at exactly eps, one ulp inside and one ulp outside; the other features equal within a
    pair (large, to widen the screen's band) and pairs 100 apart on feature 1."""
    rng = np.random.default_rng(seed)
    rows = []
    for p in range(n_pairs):
        a = rng.uniform(-50, 50, size=d).astype(np.float32)
        a[1] = np.float32(100.0 * p)
        a[0] = np.float32(rng.uniform(4.0, 7.0))
        b = a.copy()
        b[0] = np.float32(a[0] + np.float32(eps))
        b[0] = [b[0], np.nextafter(b[0], np.float32(0)), np.nextafter(b[0], np.float32(100))][p % 3]
        rows += [a, b]
    return np.array(rows, dtype=np.float32)


@pytest.mark.parametrize("d", [4, 16, 128])
def test_pairs_one_ulp_around_eps(ctx, d):
    """Decisions inside the screen's band: every pair's fate is its own label pair."""
    X = _ulp_pairs(300, d, seed=d)
    ref = _check(ctx, X, 0.75, 2)
    assert 50 < ref[2] < 300
    _, _, _, st = _fit(ctx, X, 0.75, 2, path=2 if _wg_ok(d) else 1, recheck=1)
    if _wg_ok(d):
        assert st["recheck_candidates"] > 0


def test_duplicates(ctx):
    rng = np.random.default_rng(9)
    X = np.repeat(rng.normal(size=(200, 12)).astype(np.float32) * 5, 3, axis=0)
    rng.shuffle(X)
    _check(ctx, X, 0.01, 3)
    _check(ctx, X, 0.01, 4)


# ---- parameters ----
def test_min_samples_one_makes_every_row_core(ctx):
    X = blobs(700, 16, 4, seed=3)
    ref = _check(ctx, X, 0.5, 1)
    assert ref[1].all() and (ref[0] >= 0).all()


def test_min_samples_above_n_is_all_noise(ctx):
    X = blobs(300, 16, 2, seed=4, spread=1.0)
    ref = _check(ctx, X, 100.0, 301)
    assert ref[2] == 0 and (ref[0] == -1).all() and not ref[1].any()


@pytest.mark.parametrize("d", [16, 37])
def test_cosine(ctx, d):
    rng = np.random.default_rng(d)
    C = rng.normal(size=(5, d))
    X = (C[rng.integers(0, 5, size=1000)] + 0.3 * rng.normal(size=(1000, d))) * rng.uniform(0.1, 10, size=(1000, 1))
    _check(ctx, X.astype(np.float32), 0.05, 5, metric="cosine")


# ---- structure ----
def _chain(n, eps=10.0, d=4):
    X = np.zeros((n, d), dtype=np.float32)
    X[:, 0] = 0.9 * eps * np.arange(n)
    return X


@pytest.mark.parametrize("path", [2, 1])
def test_chain_spans_every_block_and_split(ctx, path):
    """50 000 rows 0.9 eps apart: interior rows have 3 neighbours, the two ends 2, so with min_samples = 3 the chain is
    one cluster of 49 998 core rows whose two ends are border rows.  Known answer, no oracle needed."""
    n = 50000
    X = _chain(n)
    lab, core, ncl, st = _fit(ctx, X, 10.0, 3, path=path)
    assert st["last_path"] == path
    assert ncl == 1
    want_core = np.ones(n, dtype=bool)
    want_core[[0, -1]] = False
    np.testing.assert_array_equal(core, want_core)
    np.testing.assert_array_equal(lab, np.zeros(n, dtype=np.int32))


def test_chains_in_reverse_and_interleaved_order(ctx):
    """Three chains interleaved in row order: cluster ids follow each chain's lowest row, not its root history."""
    n = 3000
    X = np.zeros((3 * n, 4), dtype=np.float32)
    for c in range(3):
        X[c::3, 0] = 9.0 * np.arange(n)[::-1]
        X[c::3, 1] = 1000.0 * (2 - c)
    _check(ctx, X, 10.0, 3)


def test_border_rows_touching_two_clusters(ctx):
    """A border row exactly eps from a core row of each of two clusters takes the cluster of the lower of the two."""
    rows = []
    for k in range(40):
        y = 100.0 * k
        a = [[0.0, y], [0.25, y], [0.5, y], [1.0, y]]   # cluster A: 4 core rows at min_samples 4
        b = [[4.0, y], [4.25, y], [4.5, y], [5.0, y]]   # cluster B
        mid = [[2.5, y]]                                 # exactly 1.5 from A's 1.0 and B's 4.0: 3 neighbours, border
        rows += (mid + b + a) if k % 2 else (a + b + mid)
    X = np.array(rows, dtype=np.float32)
    X = np.concatenate([X, np.zeros((len(X), 2), dtype=np.float32)], axis=1)
    ref = _check(ctx, X, 1.5, 4)
    mids = np.array([8 if k % 2 == 0 else 0 for k in range(40)]) + 9 * np.arange(40)
    assert not ref[1][mids].any() and (ref[0][mids] >= 0).all()
    assert ref[2] == 80


# ---- passes and schedule ----
@pytest.mark.parametrize("d", [8, 64, 128])
def test_fused_equals_generic_bitwise(ctx, d):
    X = blobs(2500, d, 8, seed=50 + d, spread=4.0, std=1.0)
    eps = float(0.85 * np.sqrt(2 * d))
    out = [_fit(ctx, X, eps, 6, path=p) for p in (2, 1)]
    assert out[0][3]["last_path"] == 2 and out[1][3]["last_path"] == 1
    for a, b in zip(out[0][:3], out[1][:3]):
        np.testing.assert_array_equal(a, b)


@pytest.mark.parametrize("grid", [1, 3, 7])
def test_grid_limit_many_units_per_cta(ctx, grid):
    X = blobs(3000, 32, 6, seed=grid, spread=3.0)
    _check(ctx, X, 0.85 * 8.0, 5, grid=grid)


@pytest.mark.parametrize("n", [129, 1281, 2 * 4096 + 129])
def test_ragged_rows(ctx, n):
    X = blobs(n, 8, 5, seed=n, spread=3.0)
    _check(ctx, X, 3.4, 4)


def test_chunked_cluster_numbering(ctx):
    """More than one 4096-row chunk of the cluster numbering, with many small clusters."""
    rng = np.random.default_rng(2)
    C = rng.uniform(-1000, 1000, size=(3000, 4))
    X = (np.repeat(C, 3, axis=0) + 0.01 * rng.normal(size=(9000, 4))).astype(np.float32)
    ref = _check(ctx, X, 0.5, 3)
    assert ref[2] > 2900


# ---- errors ----
def _err(ctx, X, eps, ms, metric="euclidean"):
    with pytest.raises(_native.B2KError) as e:
        ctx.dbscan_fit(torch.from_numpy(X).cuda(), eps, ms, metric)
    return str(e.value)


def test_errors(ctx):
    X = blobs(200, 8, 2, seed=1)
    Xn = X.copy()
    Xn[17, 3] = np.nan
    assert "DBSCAN input contains NaN or infinity" in _err(ctx, Xn, 1.0, 3)
    Xi = X.copy()
    Xi[5, 0] = np.inf
    assert "DBSCAN input contains NaN or infinity" in _err(ctx, Xi, 1.0, 3)
    for eps in (0.0, -1.0, float("nan"), float("inf")):
        assert "eps" in _err(ctx, X, eps, 3)
    assert "min_samples" in _err(ctx, X, 1.0, 0)
    Xz = X.copy()
    Xz[9] = 0.0
    assert "zero row" in _err(ctx, Xz, 0.1, 3, "cosine")
    assert "no rows" in _err(ctx, X[:0], 1.0, 3)


def test_fused_path_refuses_unsupported_shapes(ctx):
    X = blobs(100, 6, 2, seed=1)
    ctx.set_option("kernel_path", 2)
    try:
        with pytest.raises(_native.B2KError, match="wgmma DBSCAN"):
            ctx.dbscan_fit(torch.from_numpy(X).cuda(), 1.0, 3)
    finally:
        ctx.set_option("kernel_path", 0)


def test_unaligned_rows_take_the_generic_pass(ctx):
    X = blobs(500, 8, 3, seed=2, spread=3.0)
    buf = torch.from_numpy(np.concatenate([np.zeros(1, np.float32), X.ravel()])).cuda()
    Xd = buf[1:].view(500, 8)
    lab, core, ncl = ctx.dbscan_fit(Xd, 1.2, 4)
    assert ctx.stats()["last_path"] == 1
    ref = do.dbscan(X, 1.2, 4)
    np.testing.assert_array_equal(lab.cpu().numpy(), ref[0])


def test_timing_and_stats(ctx):
    X = blobs(3000, 32, 6, seed=11, spread=3.0)
    ctx.set_option("time_kernels", 1)
    try:
        _, _, _, st = _fit(ctx, X, 0.85 * 8.0, 5, path=2, recheck=1)
    finally:
        ctx.set_option("time_kernels", 0)
    assert st["last_fused_ms"] > 0 and st["last_reduce_ms"] > 0 and st["last_loop_ms"] >= st["last_fused_ms"]
    assert st["recheck_rows"] > 0


# ---- estimator ----
def test_transform_of_a_local_frame_matches_the_c_abi(ctx):
    from spark_rapids_ml_b200.clustering import DBSCAN
    from spark_rapids_ml_b200.sparkshim import LocalSession

    X = blobs(3000, 16, 6, seed=21, spread=3.0)
    eps = 0.85 * np.sqrt(32)
    lab, _, _, _ = _fit(ctx, X, eps, 5)
    s = LocalSession({"spark.sql.execution.arrow.maxRecordsPerBatch": "700"})
    df = s.from_numpy(X, num_partitions=3)
    out = DBSCAN(eps=eps, min_samples=5, num_workers=1).setFeaturesCol("features").fit(df).transform(df)
    assert out.columns == df.columns + ["prediction"]
    np.testing.assert_array_equal(np.array([r["prediction"] for r in out.collect()]), lab)
    # rows matched back by a user id column that is not in row order
    ids = iter(np.random.default_rng(0).permutation(len(X)).astype(np.int64) * 7)
    dfi = df.with_appended_column("id", [[pa.array([next(ids) for _ in range(b.num_rows)], type=pa.int64())
                                          for b in p] for p in df._parts])
    out = DBSCAN(eps=eps, min_samples=5, num_workers=1, idCol="id").fit(dfi).transform(dfi)
    assert out.columns == ["features", "id", "prediction"]
    np.testing.assert_array_equal(np.array([r["prediction"] for r in out.collect()]), lab)
