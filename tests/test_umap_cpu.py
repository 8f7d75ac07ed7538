"""tests/umap_oracle.py against scikit-learn / scipy, and the hash draws (no GPU)."""
from __future__ import annotations

import numpy as np
import pytest

import umap_oracle as uo


def test_hash_draws_are_splitmix_chains():
    # splitmix64's finaliser of 0x9E3779B97F4A7C15 (seed 0), then three more rounds: fixed values, stated here so a
    # change of the chain on either side shows
    assert uo._mix(0) == 0
    h = uo.umap_hash(0, 0, 0, 0)
    assert h == uo._mix(uo._mix(uo._mix(uo._mix(0x9E3779B97F4A7C15))))
    draws = [uo.umap_hash(7, e, p, q) % 1000 for e in range(4) for p in range(50) for q in range(5)]
    assert len(set(draws)) > 600   # spread over [0, 1000)
    u = np.array([uo.unit(uo.umap_hash(1, 1 << 40, i, 0)) for i in range(20000)])
    assert 0.0 <= u.min() and u.max() < 1.0 and abs(u.mean() - 0.5) < 0.01


def test_knn_matches_sklearn():
    nn = pytest.importorskip("sklearn.neighbors")
    rng = np.random.default_rng(0)
    X = rng.normal(size=(200, 7)).astype(np.float32)
    d, i = uo.knn(X, 9)
    d2, i2 = nn.NearestNeighbors(n_neighbors=9).fit(X.astype(np.float64)).kneighbors(X.astype(np.float64))
    assert np.array_equal(i, i2)
    np.testing.assert_allclose(d, d2, rtol=1e-9, atol=1e-12)


def test_find_ab_matches_curve_fit():
    opt = pytest.importorskip("scipy.optimize")
    a, b = uo.find_ab(1.0, 0.1)
    x = np.linspace(0, 3, 300)
    y = np.where(x < 0.1, 1.0, np.exp(-(x - 0.1)))
    (a2, b2), _ = opt.curve_fit(lambda x, a, b: 1.0 / (1.0 + a * x ** (2 * b)), x, y)
    assert abs(a - a2) < 1e-6 and abs(b - b2) < 1e-6
    assert abs(a - 1.577) < 1e-3 and abs(b - 0.895) < 1e-3


def test_membership_row_sums_to_log2_k():
    rng = np.random.default_rng(1)
    X = rng.normal(size=(100, 5))
    d, i = uo.knn(X, 10)
    rho, sigma, P = uo.memberships(d, i)
    # the self edge has weight 0 and the remaining k - 1 sum to log2(k) within the bisection's tolerance
    assert np.all(P[np.arange(100), 0] == 0.0)
    np.testing.assert_allclose(P.sum(1), np.log2(10), atol=1e-4)
    np.testing.assert_allclose(rho, d[:, 1])


def test_symmetrise_union_and_intersection():
    sp = pytest.importorskip("scipy.sparse")
    rng = np.random.default_rng(2)
    n, k = 30, 4
    rows = np.repeat(np.arange(n), k)
    cols = rng.integers(0, n, n * k)
    keep = np.unique(rows * n + cols, return_index=True)[1]
    rows, cols = rows[keep], cols[keep]
    vals = rng.random(rows.size)
    A = sp.csr_matrix((vals, (rows, cols)), shape=(n, n))
    for mix in (1.0, 0.0, 0.3):
        ref = mix * (A + A.T - A.multiply(A.T)) + (1 - mix) * A.multiply(A.T)
        ref = sp.csr_matrix(ref)
        ref.eliminate_zeros()
        ref.sort_indices()
        indptr, indices, w = uo.symmetrise(rows, cols, vals, n, mix)
        assert np.array_equal(indptr, ref.indptr) and np.array_equal(indices, ref.indices)
        np.testing.assert_allclose(w, ref.data, rtol=1e-15)


def test_layout_one_epoch_does_nothing_and_schedule():
    w = np.array([1.0, 0.5, 0.001, 0.25])
    eps = uo.schedule(w, 200)
    assert np.array_equal(eps, [1.0, 2.0, np.inf, 4.0])
    Y0 = uo.random_init(4, 2, 0)
    indptr = np.array([0, 1, 2, 3, 4])
    indices = np.array([1, 0, 3, 2], np.int32)
    # no edge is due at epoch 0 (every next epoch starts at epochs_per_sample >= 1)
    assert np.array_equal(uo.layout(Y0, indptr, indices, uo.schedule(np.ones(4), 10), 10, 1, 1.5, 0.9), Y0)
    moved = uo.layout(Y0, indptr, indices, uo.schedule(np.ones(4), 10), 10, 2, 1.5, 0.9)
    assert not np.array_equal(moved, Y0)
