"""UMAP's device passes (b2k_umap_fit / b2k_umap_transform) against tests/umap_oracle.py, fed the same inputs."""
from __future__ import annotations

import numpy as np
import pytest

import umap_oracle as uo

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from spark_rapids_ml_b200 import _native  # noqa: E402

A, B = 1.5769434603113077, 0.8950608779109733   # find_ab(1.0, 0.1)


@pytest.fixture(scope="module")
def ctx():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    with _native.Context(0) as c:
        yield c


def _blobs(n, d, seed, centers=4):
    rng = np.random.default_rng(seed)
    C = rng.normal(scale=4.0, size=(centers, d))
    return (C[rng.integers(0, centers, n)] + rng.normal(size=(n, d))).astype(np.float32)


def _fit(ctx, X, **kw):
    labels = kw.pop("labels", None)
    init = kw.pop("init_array", None)
    p = _native.umap_params(a=A, b=B, **kw)
    lab = torch.from_numpy(np.asarray(labels, np.int32)).cuda() if labels is not None else None
    emb, info = ctx.umap_fit(torch.from_numpy(X).cuda(), p, labels=lab, init=init)
    return emb.cpu().numpy(), info, ctx.umap_graph(info)


def _check_graph(X, g, k, labels=None, lc=1.0, mix=1.0):
    ref = uo.graph(g["knn_dist"], g["knn_idx"], lc, mix, labels)
    np.testing.assert_allclose(g["rho"], ref["rho"], rtol=1e-12, atol=0)
    np.testing.assert_allclose(g["sigma"], ref["sigma"], rtol=1e-12, atol=0)
    assert np.array_equal(g["indptr"], ref["indptr"])
    assert np.array_equal(g["indices"], ref["indices"])
    np.testing.assert_allclose(g["weights"], ref["weights"], rtol=1e-12, atol=0)
    return ref


@pytest.mark.parametrize("d", [64, 30])
def test_graph_matches_oracle(ctx, d):
    X = _blobs(300, d, 1)
    X[10] = X[11] = X[12]            # duplicate rows
    _, info, g = _fit(ctx, X, n_neighbors=15, n_epochs=50, init="random", local_connectivity=1.5,
                      set_op_mix_ratio=0.7)
    assert ctx.stats()["last_path"] in (1, 2)
    _check_graph(X, g, 15, lc=1.5, mix=0.7)
    # the kNN itself against the fp64 oracle
    ref_d, ref_i = uo.knn(X, 15)
    np.testing.assert_allclose(g["knn_dist"], ref_d, rtol=1e-5, atol=1e-5)
    # rows, ties to the lower row: rows 10, 11 and 12 are equal, so each lists 10, 11, 12 first whatever its own index
    assert np.array_equal(g["knn_idx"], ref_i)
    assert all(list(g["knn_idx"][r, :3]) == [10, 11, 12] for r in (10, 11, 12))
    # schedule: exactly max(w) / w over the kept edges
    assert np.array_equal(g["epochs_per_sample"], uo.schedule(g["weights"], 50))


def test_graph_constant_and_k_equals_n(ctx):
    X = np.ones((40, 8), np.float32)
    _, _, g = _fit(ctx, X, n_neighbors=10, n_epochs=10, init="random")
    _check_graph(X, g, 10)
    X2 = _blobs(12, 8, 2)
    _, info, g2 = _fit(ctx, X2, n_neighbors=12, n_epochs=10, init="random")
    assert info["k"] == 12
    _check_graph(X2, g2, 12)


def test_graph_supervised_with_unknown_labels(ctx):
    X = _blobs(250, 16, 3)
    labels = np.random.default_rng(0).integers(-1, 3, 250)
    _, _, g = _fit(ctx, X, n_neighbors=10, n_epochs=20, init="random", labels=labels)
    _check_graph(X, g, 10, labels=labels)


@pytest.mark.parametrize("C", [2, 3, 16, 100])
def test_layout_epochs_match_oracle(ctx, C):
    X = _blobs(200, 32, 4)
    Y0 = uo.random_init(200, C, 99)
    dev = {}
    for E in (1, 2, 3, 4, 5):
        ctx.set_option("stop_after_epochs", E)
        try:
            dev[E], info, g = _fit(ctx, X, n_neighbors=10, n_components=C, n_epochs=30, init="given", init_array=Y0,
                                   seed=7)
        finally:
            ctx.set_option("stop_after_epochs", 0)
        assert info["epochs"] == E
    args = (g["indptr"], g["indices"], g["epochs_per_sample"], 30, 5, A, B)
    # from the same start: an fp32 layout and an fp64 one part by the rounding of close pairs, which the repulsion
    # (about 2 gamma b / 0.001 per unit of distance) amplifies each epoch; after 1 and 2 epochs they agree to 1e-3
    free = []
    uo.layout(Y0, *args, seed=7, history=free)
    for E in (1, 2):
        assert np.abs(dev[E] - free[E - 1]).max() <= 1e-3, (C, E, np.abs(dev[E] - free[E - 1]).max())
    # every epoch up to 5 from the device's own positions at its start, the schedule running on: within 1e-3
    step = []
    uo.layout(Y0, *args, seed=7, restart={e: dev[e] for e in range(1, 5)}, history=step)
    for E in range(1, 6):
        assert np.abs(dev[E] - step[E - 1]).max() <= 1e-3, (C, E, np.abs(dev[E] - step[E - 1]).max())


def test_random_init_matches_oracle(ctx):
    X = _blobs(150, 8, 5)
    ctx.set_option("stop_after_epochs", 1)
    try:
        _, info, g = _fit(ctx, X, n_neighbors=8, n_components=3, n_epochs=10, init="random", seed=123)
    finally:
        ctx.set_option("stop_after_epochs", 0)
    assert info["init_used"] == 0
    assert np.array_equal(g["init"], uo.random_init(150, 3, 123))


def test_spectral_init_against_eigsh(ctx):
    sla = pytest.importorskip("scipy.sparse.linalg")
    sp = pytest.importorskip("scipy.sparse")
    rng = np.random.default_rng(6)
    X = (rng.normal(size=(400, 8)) + np.linspace(0, 3, 400)[:, None]).astype(np.float32)
    _, info, g = _fit(ctx, X, n_neighbors=15, n_components=2, n_epochs=10, init="spectral")
    assert info["init_used"] == 1, info
    n = 400
    W = sp.csr_matrix((g["weights"], g["indices"], g["indptr"]), shape=(n, n))
    dinv = 1.0 / np.sqrt(np.asarray(W.sum(1)).ravel())
    M = sp.diags(dinv) @ W @ sp.diags(dinv)
    vals, vecs = sla.eigsh(M, k=3, which="LA", tol=1e-12)
    order = np.argsort(vals)[::-1]
    vals, vecs = vals[order][1:], vecs[:, order][:, 1:]
    np.testing.assert_allclose(g["ritz_values"], vals, atol=1e-6)
    # principal angles between the two subspaces
    Q1, _ = np.linalg.qr(g["ritz_vectors"])
    s = np.linalg.svd(Q1.T @ vecs, compute_uv=False)
    assert s.min() > 1 - 1e-6, s
    assert info["ritz_residual"] < 1e-6


def test_spectral_falls_back_on_disconnected_graph(ctx):
    X = np.concatenate([_blobs(60, 4, 7, 1), _blobs(60, 4, 8, 1) + 1000.0]).astype(np.float32)
    _, info, _ = _fit(ctx, X, n_neighbors=5, n_epochs=10, init="spectral")
    assert info["init_used"] == 0


def test_fit_bitwise_repeatable_and_grid_independent(ctx):
    X = _blobs(3000, 24, 9)
    a, _, _ = _fit(ctx, X, n_neighbors=15, n_epochs=60, init="random", seed=3)
    b, _, _ = _fit(ctx, X, n_neighbors=15, n_epochs=60, init="random", seed=3)
    ctx.set_option("grid_limit", 3)
    try:
        c, _, _ = _fit(ctx, X, n_neighbors=15, n_epochs=60, init="random", seed=3)
    finally:
        ctx.set_option("grid_limit", 0)
    assert np.array_equal(a, b) and np.array_equal(a, c)


@pytest.mark.parametrize("C", [2, 16])
def test_transform_split_equals_whole_and_nan_row(ctx, C):
    X = _blobs(1000, 16, 10)
    emb, _, _ = _fit(ctx, X, n_neighbors=15, n_components=C, n_epochs=50, init="random")
    Xt, Et = torch.from_numpy(X).cuda(), torch.from_numpy(emb).cuda()
    Q = _blobs(500, 16, 11)
    Q[7, 3] = np.nan
    p = _native.umap_params(n_neighbors=15, n_components=C, n_epochs=16, a=A, b=B, seed=5)
    whole = ctx.umap_transform(Xt, Et, torch.from_numpy(Q).cuda(), p).cpu().numpy()
    parts = np.concatenate([ctx.umap_transform(Xt, Et, torch.from_numpy(Q[s].copy()).cuda(), p).cpu().numpy()
                            for s in (slice(0, 123), slice(123, 124), slice(124, 500))])
    assert np.array_equal(np.isnan(whole), np.isnan(parts))
    assert np.array_equal(whole[~np.isnan(whole)], parts[~np.isnan(parts)])
    assert np.isnan(whole[7]).all() and np.isfinite(np.delete(whole, 7, 0)).all()
    # zero epochs: the weighted mean of the neighbours' embedding rows
    p0 = _native.umap_params(n_neighbors=15, n_components=C, n_epochs=0, a=A, b=B, seed=5)
    start = ctx.umap_transform(Xt, Et, torch.from_numpy(Q).cuda(), p0).cpu().numpy()
    for r in range(5):
        dist = np.sqrt(((X.astype(np.float64) - Q[r].astype(np.float64)) ** 2).sum(1))
        nb = np.argsort(dist, kind="stable")[:15]
        _, _, w = uo.membership_row(dist[nb].astype(np.float32), nb, -1, 1.0, 0.0, True)
        ref = (w[:, None] * emb[nb].astype(np.float64)).sum(0) / w.sum()
        assert np.abs(start[r] - ref).max() <= 1e-4


@pytest.mark.parametrize("C", [2, 16])
@pytest.mark.parametrize("gamma", [1.0, 0.0])
def test_transform_epochs_match_oracle(ctx, C, gamma):
    X = _blobs(400, 16, 14)
    emb, _, _ = _fit(ctx, X, n_neighbors=10, n_components=C, n_epochs=40, init="random", seed=2)
    Q = _blobs(60, 16, 15)
    for E in (1, 2, 5):
        p = _native.umap_params(n_neighbors=10, n_components=C, n_epochs=E, a=A, b=B, seed=9,
                                repulsion_strength=gamma)
        got = ctx.umap_transform(torch.from_numpy(X).cuda(), torch.from_numpy(emb).cuda(), torch.from_numpy(Q).cuda(),
                                 p).cpu().numpy()
        ref = uo.transform(X, emb, Q, 10, E, A, B, gamma=gamma, seed=9)
        assert np.abs(got - ref).max() <= 1e-3, (C, gamma, E, np.abs(got - ref).max())


def test_layout_without_repulsion_matches_oracle(ctx):
    # repulsion_strength = 0: negatives at d2 > 0 move nothing (the coefficient is 0, not the d2 == 0 push of 4)
    X = _blobs(200, 32, 4)
    Y0 = uo.random_init(200, 2, 99)
    ctx.set_option("stop_after_epochs", 3)
    try:
        emb, _, g = _fit(ctx, X, n_neighbors=10, n_epochs=30, init="given", init_array=Y0, seed=7,
                         repulsion_strength=0.0)
    finally:
        ctx.set_option("stop_after_epochs", 0)
    ref = uo.layout(Y0, g["indptr"], g["indices"], g["epochs_per_sample"], 30, 3, A, B, gamma=0.0, seed=7)
    assert np.abs(emb - ref).max() <= 1e-3


def test_fit_errors(ctx):
    X = _blobs(50, 4, 12)
    X[3, 1] = np.inf
    with pytest.raises(_native.B2KError, match="NaN or infinity"):
        _fit(ctx, X, n_neighbors=5, n_epochs=5, init="random")
    with pytest.raises(_native.B2KError, match="at least 2 rows"):
        _fit(ctx, np.ones((1, 4), np.float32), n_neighbors=1, n_epochs=5, init="random")
    with pytest.raises(_native.B2KError, match="n_components"):
        _fit(ctx, _blobs(50, 4, 12), n_neighbors=5, n_components=101, n_epochs=5, init="random")


@pytest.mark.slow
@pytest.mark.parametrize("C", [2, 16])
def test_layout_steady_state(ctx, C):
    X = _blobs(200_000, 32, 13, centers=20)
    a, info, _ = _fit(ctx, X, n_neighbors=15, n_components=C, n_epochs=100, init="random", seed=1)
    b, _, _ = _fit(ctx, X, n_neighbors=15, n_components=C, n_epochs=100, init="random", seed=1)
    assert info["epochs"] == 100 and np.isfinite(a).all() and np.array_equal(a, b)
