"""Random forests on one H100: every forest b2k_rf_fit grows must equal the NumPy oracle of tests/rf_oracle.py node for
node (feature, threshold bits, children, instance count, gain bits, value bits), on the cluster pass and the generic
pass, with a level split into several node groups, and under a persistent schedule squeezed onto one cluster with
flushes every tile.  k_rf_predict on the training rows must reproduce the oracle's leaves and predictions bit for bit.
Errors must be the documented ones."""
import numpy as np
import pytest

import rf_oracle as ro

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from spark_rapids_ml_b200 import _native  # noqa: E402

FUSED, GENERIC = 2, 1


@pytest.fixture(scope="module")
def ctx():
    with _native.Context(0) as c:
        yield c


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _fit(ctx, X, y, path=0, grid=0, group=0, flush=0, **kw):
    for key, v in (("kernel_path", path), ("grid_limit", grid), ("rf_group_nodes", group), ("rf_flush_tiles", flush)):
        ctx.set_option(key, v)
    try:
        out = ctx.rf_fit(_dev(X.astype(np.float32)), _dev(y.astype(np.float32)), **kw)
        return out, ctx.stats()
    finally:
        for key in ("kernel_path", "grid_limit", "rf_group_nodes", "rf_flush_tiles"):
            ctx.set_option(key, 0)


def _same(dev, ref):
    for key in ("tree_offsets", "feature", "children", "count"):
        np.testing.assert_array_equal(dev[key], ref[key], err_msg=key)
    np.testing.assert_array_equal(dev["threshold"].view(np.uint32), ref["threshold"].view(np.uint32), err_msg="threshold")
    np.testing.assert_array_equal(dev["gain"].view(np.uint64), ref["gain"].view(np.uint64), err_msg="gain")
    np.testing.assert_array_equal(dev["value"].view(np.uint64), ref["value"].view(np.uint64), err_msg="value")
    assert dev["n_values"] == ref["n_values"]


def _oracle_kw(kw):
    r = dict(kw)
    r["impurity_name"] = r.pop("impurity", "gini")
    r["features_per_node"] = r.get("features_per_node") or 0
    return r


def _check(ctx, X, y, paths=(FUSED, GENERIC), **kw):
    ref = ro.fit(X, y, **_oracle_kw(kw))
    for path in paths:
        dev, st = _fit(ctx, X, y, path=path, **kw)
        assert st["last_path"] == path
        _same(dev, ref)
    return ref


def data(n, d, C, seed, absent=()):
    rng = np.random.default_rng(seed)
    X = rng.normal(size=(n, d)).astype(np.float32)
    X[:, : max(1, d // 4)] = np.round(X[:, : max(1, d // 4)] * 4) / 4   # some features with few values
    s = X[:, 0] + (X[:, 1] if d > 1 else 0) + 0.7 * rng.normal(size=n)
    y = np.floor((s - s.min()) / (s.max() - s.min() + 1e-9) * C).astype(np.int64)
    for a in absent:
        y[y == a] = (a + 1) % C
    y[0] = C - 1   # the class count is max label + 1
    return X, y.astype(np.float32)


@pytest.mark.parametrize("d", [1, 3, 17, 128, 512])
def test_feature_counts(ctx, d):
    X, y = data(1500, d, 2, seed=d)
    _check(ctx, X, y, n_trees=4, max_depth=5, max_bins=32, features_per_node=ro.features_per_node("sqrt", d, 4, True),
           seed=11)


@pytest.mark.parametrize("C, absent", [(2, ()), (3, (1,)), (10, (2, 7)), (64, (5, 6, 40))])
def test_classes(ctx, C, absent):
    X, y = data(3000, 12, C, seed=C, absent=absent)
    _check(ctx, X, y, n_trees=3, max_depth=6, max_bins=32, features_per_node=4, seed=5)


@pytest.mark.parametrize("max_bins", [2, 32, 256])
@pytest.mark.parametrize("impurity", ["gini", "entropy"])
def test_bins_and_impurity(ctx, max_bins, impurity):
    X, y = data(4000, 9, 3, seed=max_bins)
    _check(ctx, X, y, n_trees=3, max_depth=5, max_bins=max_bins, features_per_node=3, impurity=impurity, seed=3)


@pytest.mark.parametrize("max_depth", [0, 1, 5, 12])
def test_depths(ctx, max_depth):
    X, y = data(2500, 8, 4, seed=21)
    _check(ctx, X, y, n_trees=2, max_depth=max_depth, max_bins=32, features_per_node=8, seed=9)


@pytest.mark.parametrize("n_trees", [1, 20, 100])
@pytest.mark.parametrize("bootstrap", [True, False])
def test_tree_counts_and_bootstrap(ctx, n_trees, bootstrap):
    X, y = data(800, 6, 2, seed=n_trees)
    _check(ctx, X, y, n_trees=n_trees, max_depth=4, max_bins=16, features_per_node=2, bootstrap=bootstrap, seed=13)


@pytest.mark.parametrize("strategy", ["auto", "all", "sqrt", "log2", "onethird", "3", "0.4"])
def test_subset_strategies(ctx, strategy):
    X, y = data(1200, 20, 3, seed=4)
    k = ro.features_per_node(strategy, 20, 5, True)
    _check(ctx, X, y, n_trees=5, max_depth=4, max_bins=32, features_per_node=k, seed=17)


def test_edge_data(ctx):
    X, y = data(1000, 6, 3, seed=8)
    X[:, 2] = 3.5                                    # a constant feature
    X[500:] = X[:500]                                # duplicate rows
    y[500:] = y[:500]
    _check(ctx, X, y, n_trees=4, max_depth=6, max_bins=32, features_per_node=3, seed=1)
    _check(ctx, X, np.zeros_like(y), n_trees=2, max_depth=4, max_bins=32, features_per_node=3, seed=1)   # one class
    _check(ctx, X, y, n_trees=2, max_depth=8, max_bins=32, features_per_node=6, min_instances=150, seed=2)
    _check(ctx, X, y, n_trees=2, max_depth=8, max_bins=32, features_per_node=6, min_info_gain=0.05, seed=2)
    _check(ctx, X[:, [2]], y, n_trees=2, max_depth=3, max_bins=32, features_per_node=1, seed=2)   # nothing to split


@pytest.mark.parametrize("span", ["wide", "constant", "small"])
def test_regression(ctx, span):
    rng = np.random.default_rng(5)
    X = rng.normal(size=(3000, 10)).astype(np.float32)
    if span == "wide":
        y = np.sign(X[:, 0]) * 10.0 ** (X[:, 1] * 1.5).clip(-3, 3)
    elif span == "constant":
        y = np.full(3000, 2.5)
    else:
        y = 1e-3 * (X[:, 0] - X[:, 2] ** 2 + 0.1 * rng.normal(size=3000))
    ref = _check(ctx, X, y.astype(np.float32), n_trees=5, max_depth=6, max_bins=32, features_per_node=4,
                 impurity="variance", seed=7)
    if span == "constant":
        assert ref["tree_offsets"][-1] == 5


def test_regression_deep_many_trees(ctx):
    rng = np.random.default_rng(6)
    X = rng.normal(size=(2000, 16)).astype(np.float32)
    y = (X[:, 0] * 3 + np.sin(X[:, 1] * 2) + 0.2 * rng.normal(size=2000)).astype(np.float32)
    _check(ctx, X, y, n_trees=20, max_depth=12, max_bins=64, features_per_node=6, impurity="variance", seed=4)


@pytest.mark.parametrize("impurity", ["gini", "variance"])
def test_node_groups_and_steady_state(ctx, impurity):
    """A level forced into groups of 1 and 3 nodes, and the cluster pass on one cluster flushing every 1 / 2 tiles per
    CTA (hundreds of tiles, many flush rounds), all equal the one-group forest."""
    X, y = data(20000, 8, 3, seed=2)
    if impurity == "variance":
        y = (X[:, 0] * 2 + X[:, 3]).astype(np.float32)
    kw = dict(n_trees=6, max_depth=6, max_bins=32, features_per_node=3, impurity=impurity, seed=8)
    ref = ro.fit(X, y, **_oracle_kw(kw))
    base, st = _fit(ctx, X, y, path=FUSED, **kw)
    _same(base, ref)
    for opts in (dict(group=1), dict(group=3), dict(group=3, path=GENERIC), dict(grid=8, flush=1),
                 dict(grid=8, flush=2), dict(grid=16, flush=3, group=5)):
        dev, st2 = _fit(ctx, X, y, **{"path": FUSED, **opts}, **kw)
        _same(dev, ref)
        if opts.get("group"):
            assert st2["recheck_rows"] > st["recheck_rows"], opts   # more histogram passes


def test_generic_pass_by_shape(ctx):
    """A node histogram larger than the cluster (d = 512, all features, 256 bins, 10 classes) takes the generic pass;
    forcing the cluster pass is an error."""
    X, y = data(600, 512, 10, seed=3)
    X[:, :] = np.random.default_rng(1).normal(size=X.shape)
    kw = dict(n_trees=1, max_depth=2, max_bins=256, features_per_node=512, seed=1)
    ref = ro.fit(X, y, **_oracle_kw(kw))
    dev, st = _fit(ctx, X, y, **kw)
    assert st["last_path"] == GENERIC
    _same(dev, ref)
    with pytest.raises(_native.B2KError) as e:
        _fit(ctx, X, y, path=FUSED, **kw)
    assert e.value.code == 4


@pytest.mark.parametrize("classification", [True, False])
def test_predict_reproduces_oracle(ctx, classification):
    X, y = data(5000, 12, 4, seed=12)
    if not classification:
        y = (X[:, 0] - X[:, 5] * 0.5).astype(np.float32)
    kw = dict(n_trees=20, max_depth=7, max_bins=32, features_per_node=4,
              impurity="gini" if classification else "variance", seed=3)
    dev, _ = _fit(ctx, X, y, **kw)
    ref = ro.fit(X, y, **_oracle_kw(kw))
    _same(dev, ref)
    raw, prob, pred = ctx.rf_predict(_dev(X), dev, classification)
    r_raw, r_prob, r_pred = ro.predict(X, ref, classification)
    np.testing.assert_array_equal(pred.cpu().numpy().view(np.uint64), r_pred.view(np.uint64))
    if classification:
        np.testing.assert_array_equal(raw.cpu().numpy().view(np.uint64), r_raw.view(np.uint64))
        np.testing.assert_array_equal(prob.cpu().numpy().view(np.uint64), r_prob.view(np.uint64))
        # a forest too large for shared memory walks the nodes through L1/L2
        big = dict(kw, n_trees=100, max_depth=10)
        devb, _ = _fit(ctx, X, y, **big)
        assert devb["tree_offsets"][-1] * 16 > 48 * 1024
        _, _, pb = ctx.rf_predict(_dev(X), devb, True)
        np.testing.assert_array_equal(pb.cpu().numpy(), ro.predict(X, devb, True)[2])


@pytest.mark.parametrize("kw, code, msg", [
    (dict(max_depth=-1), 1, "maxDepth given invalid value -1"),
    (dict(max_bins=-1), 1, "maxBins given invalid value -1"),
    (dict(max_bins=257), 1, "maxBins given invalid value 257"),
    (dict(max_depth=17), 4, "maxDepth 17 > 16"),
    (dict(n_trees=0), 1, "numTrees given invalid value 0"),
    (dict(min_instances=0), 1, "minInstancesPerNode"),
    (dict(min_info_gain=-1.0), 1, "minInfoGain"),
    (dict(features_per_node=9), 1, "features per node"),
])
def test_param_errors(ctx, kw, code, msg):
    X, y = data(100, 8, 2, seed=1)
    with pytest.raises(_native.B2KError) as e:
        _fit(ctx, X, y, **kw)
    assert e.value.code == code and msg in str(e.value), str(e.value)


def test_data_errors(ctx):
    X, y = data(100, 4, 2, seed=1)
    for bad_X, bad_y, msg in ((np.nan, None, "NaN or infinity"), (None, np.inf, "NaN or infinity"),
                              (None, 1.5, "Labels MUST be Integers"), (None, -1.0, "Labels MUST be in")):
        Xb, yb = X.copy(), y.copy()
        if bad_X is not None:
            Xb[3, 1] = bad_X
        if bad_y is not None:
            yb[4] = bad_y
        with pytest.raises(_native.B2KError) as e:
            _fit(ctx, Xb, yb)
        assert msg in str(e.value), str(e.value)
    with pytest.raises(_native.B2KError) as e:
        _fit(ctx, X[:0], y[:0])
    assert "empty partition" in str(e.value)
