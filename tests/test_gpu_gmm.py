"""The Gaussian mixture passes on the device (b2k_gmm_fit / b2k_gmm_predict) against the fp64 oracle tests/gmm_oracle.py:
the E pass on both paths over widths, component counts, a rank-deficient component and offset data; the wgmma E pass
past one turn of its ring with many tiles per CTA; full fits from injected parameters; bitwise repeatability; every
error path.

Tolerances (DESIGN §22): the generic E pass is fp64 throughout, so its responsibilities match the oracle to ~1e-9.  The
wgmma pass forms P_k (x - c) in 3xTF32 from x - c rounded once to fp32, a relative error of a few 1e-7 in each
whitened coordinate, so q_ik carries an absolute error of about 1e-6 (1 + q_ik) and a responsibility moves by at most
that much; the log-likelihood by the sum over rows."""
import ctypes

import numpy as np
import pytest
import torch

import gmm_oracle as go
from spark_rapids_ml_b200 import _native

pytestmark = pytest.mark.gpu


def _mixture(n, d, k, seed, shift=0.0):
    rng = np.random.default_rng(seed)
    means = rng.normal(scale=4.0, size=(k, d))
    z = rng.integers(0, k, size=n)
    X = means[z] + rng.normal(size=(n, d)) * rng.uniform(0.5, 1.5, size=(k, d))[z] + shift
    return X.astype(np.float32)


def _model(X, k, seed, rank_deficient=False):
    """A model near the data: means of k rows, covariances of random spd matrices; component 0 rank-deficient."""
    rng = np.random.default_rng(seed)
    d = X.shape[1]
    Xd = X.astype(np.float64)
    mu = Xd[rng.choice(len(X), k, replace=False)]
    cov = np.empty((k, d, d))
    for j in range(k):
        A = rng.normal(size=(d, d)) / np.sqrt(d)
        cov[j] = A @ A.T + np.eye(d) * rng.uniform(0.5, 2.0)
    if rank_deficient and d > 1:
        B = rng.normal(size=(d, max(1, d // 2)))
        cov[0] = B @ B.T
    w = rng.uniform(0.5, 1.5, size=k)
    return w / w.sum(), mu, cov


def _dev(X):
    return torch.from_numpy(np.ascontiguousarray(X)).cuda()


CASES = [(1, 2), (3, 2), (4, 2), (4, 64), (128, 2), (128, 64), (130, 2), (256, 2), (3, 65), (256, 65)]


@pytest.mark.parametrize("path", [_native.PATH_AUTO, _native.PATH_GENERIC])
@pytest.mark.parametrize("d,k", CASES)
def test_e_pass_matches_oracle(d, k, path):
    n = 700 if d < 256 else 300
    X = _mixture(n, d, min(k, 8), seed=d * 1000 + k, shift=0.0)
    w, mu, cov = _model(X, k, seed=d + k, rank_deficient=True)
    r_ref, ll_ref, lab_ref = go.e_step(X, w, mu, cov)
    wg_shape = d % 4 == 0 and 4 <= d <= 128 and k <= 64
    with _native.Context(0) as ctx:
        ctx.set_option("kernel_path", path)
        prob, lab = ctx.gmm_predict(_dev(X), w, mu, cov)
        st = ctx.stats()
        fit = ctx.gmm_fit(_dev(X), k, init=(w, mu, cov), max_iter=1, tol=0.0)
    assert st["last_path"] == (_native.PATH_FUSED if wg_shape and path == _native.PATH_AUTO else _native.PATH_GENERIC)
    prob = prob.cpu().numpy()
    tol = 1e-9 if st["last_path"] == _native.PATH_GENERIC else 2e-4
    np.testing.assert_allclose(prob, r_ref, atol=tol, rtol=0)
    np.testing.assert_allclose(prob.sum(axis=1), 1.0, atol=1e-12)
    lab = lab.cpu().numpy()
    close = np.sort(r_ref, axis=1)[:, -1] - np.sort(r_ref, axis=1)[:, -2] > 2 * tol
    np.testing.assert_array_equal(lab[close], lab_ref[close])
    assert abs(fit["log_likelihood"] - ll_ref) <= (1e-9 if tol < 1e-6 else 1e-4) * (abs(ll_ref) + n), \
        (fit["log_likelihood"], ll_ref)


@pytest.mark.parametrize("path", [_native.PATH_AUTO, _native.PATH_GENERIC])
def test_offset_data(path):
    X = _mixture(2000, 8, 3, seed=5, shift=1.0e4)
    w, mu, cov = _model(X, 3, seed=6)
    r_ref, ll_ref, _ = go.e_step(X, w, mu, cov)
    with _native.Context(0) as ctx:
        ctx.set_option("kernel_path", path)
        prob, _ = ctx.gmm_predict(_dev(X), w, mu, cov)
        fit = ctx.gmm_fit(_dev(X), 3, init=(w, mu, cov), max_iter=1, tol=0.0)
    np.testing.assert_allclose(prob.cpu().numpy(), r_ref, atol=2e-4 if path == _native.PATH_AUTO else 1e-9)
    assert abs(fit["log_likelihood"] - ll_ref) <= 1e-4 * abs(ll_ref)


def test_wgmma_past_one_turn_of_the_ring():
    # 2 CTAs over 60 tiles of 128 rows: each CTA runs 30 units of 40 blocks through the 2-stage ring
    X = _mixture(128 * 60 - 5, 64, 6, seed=7)
    w, mu, cov = _model(X, 40, seed=8)
    r_ref, _, _ = go.e_step(X, w, mu, cov)
    with _native.Context(0) as ctx:
        ctx.set_option("grid_limit", 2)
        prob, _ = ctx.gmm_predict(_dev(X), w, mu, cov)
        assert ctx.stats()["last_path"] == _native.PATH_FUSED
    np.testing.assert_allclose(prob.cpu().numpy(), r_ref, atol=2e-4)


@pytest.mark.parametrize("d,k", [(64, 3), (132, 2)])
def test_weighted_gram_past_one_turn_of_the_ring(d, k):
    # one M step from an injected model, so the E step is the same on both paths and the M passes are compared: with
    # grid_limit = 1 the wgmma Gram pass runs one CTA per (component, tile) over 20 row ranges of 128 chunks each through
    # its 3-slot ring; d = 132 has two feature blocks (an off-diagonal tile) and runs the generic E pass
    X = _mixture(4096 * 20 - 7, d, k, seed=14, shift=3.0)
    w, mu, cov = _model(X, k, seed=15)
    r, _, _ = go.e_step(X, w, mu, cov)
    w1, mu1, cov1 = go.m_step(X, r)
    outs = {}
    for path in (_native.PATH_AUTO, _native.PATH_GENERIC):
        with _native.Context(0) as ctx:
            ctx.set_option("kernel_path", path)
            ctx.set_option("grid_limit", 1)
            ctx.reset_stats()
            outs[path] = ctx.gmm_fit(_dev(X), k, init=(w, mu, cov), max_iter=1, tol=0.0)
            outs[path]["stats"] = ctx.stats()
    assert outs[_native.PATH_AUTO]["stats"]["fused_tc_launches"] >= 1
    assert outs[_native.PATH_GENERIC]["stats"]["fused_tc_launches"] == 0
    scale = np.abs(cov1).max()
    for path, atol in ((_native.PATH_GENERIC, 1e-9), (_native.PATH_AUTO, 1e-4)):
        o = outs[path]
        np.testing.assert_allclose(o["weights"], w1, atol=atol)
        np.testing.assert_allclose(o["means"], mu1, atol=atol * 10)
        np.testing.assert_allclose(o["covs"], cov1, atol=atol * scale)


@pytest.mark.parametrize("path", [_native.PATH_AUTO, _native.PATH_GENERIC])
def test_fit_matches_oracle_em(path):
    X = _mixture(3000, 4, 3, seed=9, shift=50.0)
    w0, mu0, cov0 = go.random_init(X, 3, 21)
    w, mu, cov, ll, it, _ = go.fit(X, w0, mu0, cov0, 8, 0.0)
    with _native.Context(0) as ctx:
        ctx.set_option("kernel_path", path)
        out = ctx.gmm_fit(_dev(X), 3, init=(w0, mu0, cov0), max_iter=8, tol=0.0)
        out2 = ctx.gmm_fit(_dev(X), 3, max_iter=8, tol=0.0, seed=21)
    assert out["n_iter"] == it == 8
    atol = 1e-8 if path == _native.PATH_GENERIC else 1e-3
    np.testing.assert_allclose(out["weights"], w, atol=atol)
    np.testing.assert_allclose(out["means"], mu, atol=atol * 10)
    np.testing.assert_allclose(out["covs"], cov, atol=atol * 10)
    assert abs(out["log_likelihood"] - ll) <= atol * abs(ll)
    assert out["cluster_sizes"].sum() == 3000
    # the seeded start is the oracle's rule
    for key in ("weights", "means", "covs", "log_likelihood"):
        np.testing.assert_array_equal(out2[key], out[key])


def test_tolerance_stops_and_max_iter_zero():
    X = _mixture(2000, 4, 2, seed=10)
    with _native.Context(0) as ctx:
        a = ctx.gmm_fit(_dev(X), 2, max_iter=200, tol=0.01, seed=3)
        z = ctx.gmm_fit(_dev(X), 2, max_iter=0, seed=3)
    assert 2 <= a["n_iter"] < 200
    assert z["n_iter"] == 0 and z["log_likelihood"] == -np.inf
    w0, mu0, cov0 = go.random_init(X, 2, 3)
    np.testing.assert_array_equal(z["means"], mu0)
    np.testing.assert_array_equal(z["covs"], cov0)


@pytest.mark.parametrize("d,k", [(16, 4), (20, 3)])
def test_two_calls_are_bitwise_equal(d, k):
    X = _mixture(5000, d, k, seed=11)
    with _native.Context(0) as ctx:
        a = ctx.gmm_fit(_dev(X), k, max_iter=5, tol=0.0, seed=4)
        b = ctx.gmm_fit(_dev(X), k, max_iter=5, tol=0.0, seed=4)
        pa_, la = ctx.gmm_predict(_dev(X), a["weights"], a["means"], a["covs"])
        pb, lb = ctx.gmm_predict(_dev(X), a["weights"], a["means"], a["covs"])
    for key in ("weights", "means", "covs", "cluster_sizes"):
        np.testing.assert_array_equal(a[key], b[key])
    assert a["log_likelihood"] == b["log_likelihood"]
    assert torch.equal(pa_, pb) and torch.equal(la, lb)
    np.testing.assert_array_equal(np.bincount(la.cpu().numpy(), minlength=k), a["cluster_sizes"])


def test_error_paths():
    X = _mixture(100, 3, 2, seed=12)
    w, mu, cov = _model(X, 2, seed=13)
    with _native.Context(0) as ctx:
        def err(fn, code, msg):
            with pytest.raises(_native.B2KError) as e:
                fn()
            assert e.value.code == code and msg in str(e.value), str(e.value)

        err(lambda: ctx.gmm_fit(_dev(X), 1), 1, "k must be > 1")
        err(lambda: ctx.gmm_fit(_dev(X[:5]), 6), 1, "exceeds the 5 rows")
        err(lambda: ctx.gmm_fit(_dev(X), 2, max_iter=-1), 1, "maxIter")
        err(lambda: ctx.gmm_fit(_dev(X), 2, tol=-1.0), 1, "tol")
        err(lambda: ctx.gmm_fit(_dev(np.zeros((10, 257), np.float32)), 2), 4, "got d = 257, k = 2")
        err(lambda: ctx.gmm_fit(_dev(np.zeros((300, 4), np.float32)), 257), 4, "got d = 4, k = 257")
        err(lambda: ctx.gmm_predict(_dev(np.zeros((10, 257), np.float32)), [0.5, 0.5], np.zeros((2, 257)),
                                    np.stack([np.eye(257)] * 2)), 4, "got d = 257, k = 2")
        # the C entry point's own argument checks: d < 1 and an unknown init mode
        out = [np.zeros(64) for _ in range(3)]
        ll, it, sizes = ctypes.c_double(), ctypes.c_int(), np.zeros(2, dtype=np.int64)
        Xd = _dev(X)

        def raw(d, mode):
            return lambda: ctx._check(ctx._L.b2k_gmm_fit(
                ctx._h, Xd.data_ptr(), 100, d, 2, mode, None, None, None, 3, 0.0, 0, out[0].ctypes.data,
                out[1].ctypes.data, out[2].ctypes.data, ctypes.byref(ll), ctypes.byref(it), sizes.ctypes.data,
                ctx._stream()))

        err(raw(0, _native.INIT_RANDOM), 1, "d must be >= 1")
        err(raw(3, _native.INIT_KMEANS_PARALLEL), 1, "init_mode must be")
        err(raw(3, _native.INIT_ARRAY), 1, "B2K_INIT_ARRAY needs")
        Xn = X.copy()
        Xn[7, 1] = np.nan
        err(lambda: ctx.gmm_fit(_dev(Xn), 2, max_iter=3), 1, "NaN or an infinity")
        Xi = X.copy()
        Xi[3, 0] = np.inf
        err(lambda: ctx.gmm_fit(_dev(Xi), 2, max_iter=3), 1, "NaN or an infinity")
        cz = cov.copy()
        cz[1] = 0.0
        err(lambda: ctx.gmm_fit(_dev(X), 2, init=(w, mu, cz), max_iter=3), 1, "no eigenvalue above the tolerance")
        err(lambda: ctx.gmm_predict(_dev(X), w, mu, cz), 1, "no eigenvalue above the tolerance")
        err(lambda: ctx.gmm_fit(_dev(np.ones((20, 3), np.float32)), 2, max_iter=3), 1,
            "no eigenvalue above the tolerance")
        ctx.set_option("kernel_path", _native.PATH_FUSED)
        err(lambda: ctx.gmm_predict(_dev(X), w, mu, cov), 4, "wgmma E pass")
        err(lambda: ctx.gmm_fit(_dev(X), 2, max_iter=2), 4, "on every rank")
        # the context stays usable after every error
        ctx.set_option("kernel_path", _native.PATH_AUTO)
        out = ctx.gmm_fit(_dev(X), 2, max_iter=2)
    assert out["n_iter"] == 2
