"""The fp64 Gram passes of b2k_gram.cu held to fp64 oracles entry by entry.

Unweighted pass (W = false), through Context.linreg_moments: its [d][d] block is the Gram of the rows centred on
mu32 = fl32(mean), unpacked by k_gram_unpack, less n delta delta^T (delta = mean - mu32) on the host.  kernel_path 2
forces the wgmma pass, 1 the generic one, and grid_limit caps the wgmma CTAs, so the P CTAs of one tile take
ceil(nrange / P) or floor(nrange / P) of the 4096-row ranges.  The oracle restates that block in fp64 on the device
from the float32 rows and the returned mean.

Weighted pass (W = true), through Context.gmm_fit(init=(w, mu, Sigma), max_iter=1, tol=0) at shapes where the E pass is
the fp64 generic one (d > 128, or k >= 65): kernel_path AUTO (wgmma Gram) and GENERIC read the same responsibilities bit
for bit, and k_gmm_mom is the same kernel on the same input, so the weights and means agree exactly and the covariances
differ by the Gram pass alone.  The generic fit is also held to gmm_oracle.m_step in fp64 on the responsibilities of the
generic predict pass for the same model.

Bounds, entry by entry, from the kernels' arithmetic:
- Generic pass, W = false: x - mu is rounded once to fp32 (2^-24 relative in each operand), then multiplied and summed
  in fp64: |G - G_ref| <= (2^-23 + n 2^-53) sum_rows |v_i v_j|, v = x - mu32 (linear regression's rule).
- wgmma pass: eps_wg sum_rows |v_i v_j|, with eps_wg the sum of
    fp32 centring                                          2^-23     (2^-24 in each operand)
    tf32 split, v = hi + lo + O(2^-22 v), lo.lo dropped     3 2^-22
    12 truncating wgmma accumulations per 32-row chunk     12 2^-23
    GW_RANGE / GW_KC = 128 rounded fp32 chunk additions    128 2^-24
  = 83 2^-23 (about 9.9e-6), plus n 2^-53 for the fp64 flushes and the fold.
- Weighted, per component k and entry (a, b): the same form relative to the component's own spread,
    |Sigma_k - Sigma_k'| <= eps S^abs_k,  S^abs_k = sum_i r_ik |x_i - mu_k|_a |x_i - mu_k|_b / N_k,
  with S^abs_k from the oracle's responsibilities and means.  The wgmma pass adds the row weight's rounding to eps_wg:
  fl32 of the weight (2^-24), its square root rounded (2^-24 in each operand) and the scaled value rounded (2^-24 in
  each operand), 5 2^-24 in all; the generic pass's own n 2^-53 is added on both sides of the difference.  The generic
  fit against the oracle: the E passes of fit and predict agree to the last bits, so 1e-9 S^abs_k.
A component whose covariance is wrong by more than that relative to its own spread fails, however small it is.
Each test prints the observed worst ratio to its bound.
"""
import numpy as np
import pytest
import torch

import gmm_oracle as go
from _ranks_child_gmm import dead_component
from spark_rapids_ml_b200 import _native

pytestmark = pytest.mark.gpu

EPS_GEN = 2.0 ** -23
EPS_WG = 83 * 2.0 ** -23
EPS_W = EPS_WG + 5 * 2.0 ** -24
RANGE = 4096


# ---------------------------------------------------------------------------------------------------------------------
# unweighted pass
# ---------------------------------------------------------------------------------------------------------------------
def _rows(n, d, seed, mixed=False):
    rng = np.random.default_rng(seed)
    X = rng.normal(size=(n, d)) + rng.normal(size=d)
    if mixed:
        # columns from 1e-3 to 1e3, every third one offset by 1e3: the small ones are invisible to a max-entry bound
        X = X * np.logspace(-3, 3, d) + np.where(np.arange(d) % 3 == 1, 1e3, 0.0)
    y = rng.normal(size=n)
    return X.astype(np.float32), y.astype(np.float32)


def _moments(ctx, Xd, yd, path, grid_limit=0):
    ctx.set_option("kernel_path", path)
    ctx.set_option("grid_limit", grid_limit)
    try:
        n, mean, M = ctx.linreg_moments(Xd, yd)
        last = ctx.stats()["last_path"]
    finally:
        ctx.set_option("kernel_path", _native.PATH_AUTO)
        ctx.set_option("grid_limit", 0)
    return n, mean, M, last


def _check_gram(Xd, mean, M, eps, what):
    """M[:d, :d] against the fp64 Gram about mu32 less n delta delta^T, entry by entry; returns the worst ratio."""
    n, d = Xd.shape
    mu32 = torch.from_numpy(mean[:d].astype(np.float32).astype(np.float64)).cuda()
    delta = torch.from_numpy(mean[:d]).cuda() - mu32
    V = Xd.double() - mu32   # exact: the difference of two floats
    A = V.abs()
    G_ref = (V.T @ V - n * torch.outer(delta, delta)).cpu().numpy()
    S = (A.T @ A).cpu().numpy()
    G = M[:d, :d]
    bound = (eps + n * 2.0 ** -53) * S + 2.0 ** -52 * n * np.abs(np.outer(delta.cpu().numpy(), delta.cpu().numpy()))
    err = np.abs(G - G_ref)
    ratio = float((err / np.where(bound > 0, bound, 1.0)).max())
    print(f"{what}: worst |G - G_ref| / bound = {ratio:.3g}")
    bad = np.argwhere(err > bound)
    assert bad.size == 0, (what, len(bad), bad[:5].tolist(), [(G[i, j], G_ref[i, j], bound[i, j]) for i, j in bad[:5]])
    assert np.array_equal(M, M.T), what
    return ratio


def _both_paths(X, y, grid_limits=(0,), what=""):
    n, d = X.shape
    Xd, yd = torch.from_numpy(X).cuda(), torch.from_numpy(y).cuda()
    with _native.Context(0) as ctx:
        nn, mean, M, last = _moments(ctx, Xd, yd, _native.PATH_GENERIC)
        assert nn == n and last == _native.PATH_GENERIC
        np.testing.assert_allclose(mean[:d], X.astype(np.float64).mean(0), rtol=1e-12,
                                   atol=1e-12 * float(np.abs(X).max()))
        _check_gram(Xd, mean, M, EPS_GEN, f"{what} generic")
        if d % 4 == 0:
            for g in grid_limits:
                _, mean2, M2, last = _moments(ctx, Xd, yd, _native.PATH_FUSED, g)
                assert last == _native.PATH_FUSED
                assert np.array_equal(mean2, mean)
                _check_gram(Xd, mean2, M2, EPS_WG, f"{what} wgmma grid_limit={g}")


WG_WIDTHS = [4, 8, 32, 36, 124, 128, 132, 256, 260, 1020, 1024]
ROWS = [2, 31, 33, RANGE, RANGE + 1, 3 * RANGE + 5]


@pytest.mark.parametrize("n", ROWS)
@pytest.mark.parametrize("d", WG_WIDTHS)
def test_unweighted_wgmma_widths_and_rows(d, n):
    # partial 32-feature boxes (d = 4, 8, 36, 260), ragged off-diagonal blocks (132, 260, 1020) and 36 tiles (1024);
    # one row, a partial chunk, a partial range, one row past a range
    X, y = _rows(n, d, seed=d * 7 + n)
    _both_paths(X, y, what=f"d={d} n={n}")


@pytest.mark.parametrize("d,n", [(256, 4 * RANGE + 1), (36, 3 * RANGE + 5), (132, 5 * RANGE + 100),
                                 (1024, 2 * RANGE + 3)])
def test_unweighted_grid_limits(d, n):
    # d = 256, n = 4 * 4096 + 1, grid_limit = 7: 3 tiles, P = 2 over 5 ranges, so the CTAs of a tile take 3 and 2 ranges
    X, y = _rows(n, d, seed=d + n)
    _both_paths(X, y, grid_limits=(0, 1, 2, 7), what=f"d={d} n={n}")


@pytest.mark.parametrize("n", [33, 65])
@pytest.mark.parametrize("d", [1, 3, 5, 31, 33, 129, 1023])
def test_unweighted_generic_widths(d, n):
    # 2 and 3 row spans of 17 and 22 rows: span_rows is not a multiple of the 32-row staging block
    X, y = _rows(n, d, seed=d * 3 + n)
    Xd, yd = torch.from_numpy(X).cuda(), torch.from_numpy(y).cuda()
    with _native.Context(0) as ctx:
        _, mean, M, last = _moments(ctx, Xd, yd, _native.PATH_AUTO)
    assert last == _native.PATH_GENERIC
    _check_gram(Xd, mean, M, EPS_GEN, f"generic d={d} n={n}")


@pytest.mark.parametrize("d,n", [(64, 20000), (260, 3 * RANGE + 5), (33, 5000)])
def test_unweighted_mixed_scales(d, n):
    X, y = _rows(n, d, seed=d, mixed=True)
    _both_paths(X, y, grid_limits=(0, 2), what=f"mixed d={d} n={n}")


def test_unweighted_unaligned_rows_take_the_generic_pass():
    # the other passes of b2k_moments_impl (k_colsum, k_xty) read X with scalar loads, so a view 4 bytes past a 16-byte
    # boundary is legal input; the wgmma pass's TMA map needs 16-byte alignment and is not taken
    n, d = 5000, 64
    X, y = _rows(n, d, seed=5)
    buf = torch.from_numpy(np.concatenate([np.zeros(1, np.float32), X.reshape(-1)])).cuda()
    Xu = buf[1:].view(n, d)
    assert Xu.data_ptr() % 16 == 4
    Xa, yd = torch.from_numpy(X).cuda(), torch.from_numpy(y).cuda()
    with _native.Context(0) as ctx:
        _, mean, M, last = _moments(ctx, Xu, yd, _native.PATH_AUTO)
        assert last == _native.PATH_GENERIC
        _, mean_a, M_a, last_a = _moments(ctx, Xa, yd, _native.PATH_GENERIC)
        with pytest.raises(_native.B2KError, match="16-byte aligned"):
            _moments(ctx, Xu, yd, _native.PATH_FUSED)
    assert last_a == _native.PATH_GENERIC
    assert np.array_equal(mean, mean_a) and np.array_equal(M, M_a)
    _check_gram(Xu, mean, M, EPS_GEN, "unaligned")


@pytest.mark.parametrize("path,grid_limit", [(_native.PATH_FUSED, 7), (_native.PATH_FUSED, 0),
                                             (_native.PATH_GENERIC, 0)])
def test_unweighted_two_calls_are_bitwise_equal(path, grid_limit):
    X, y = _rows(4 * RANGE + 1, 256, seed=9)
    Xd, yd = torch.from_numpy(X).cuda(), torch.from_numpy(y).cuda()
    with _native.Context(0) as ctx:
        a = _moments(ctx, Xd, yd, path, grid_limit)
        b = _moments(ctx, Xd, yd, path, grid_limit)
    assert a[3] == b[3] == path
    assert np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])
    assert np.array_equal(a[2], a[2].T)


# ---------------------------------------------------------------------------------------------------------------------
# weighted pass
# ---------------------------------------------------------------------------------------------------------------------
def _truth(n, d, k, seed, s=0.05, shift=1.0):
    """Rows of k diagonal Gaussians and their parameters.  Spreads are scaled by s: with MLlib's + EPS, a density below
    2.2e-16 (unit variances at d >= 128) would make every responsibility 1 / k."""
    rng = np.random.default_rng(seed)
    means = s * rng.normal(scale=4.0, size=(k, d)) + shift
    sd = s * rng.uniform(0.5, 1.5, size=(k, d))
    z = np.arange(n) % k
    X = (means[z] + rng.normal(size=(n, d)) * sd[z]).astype(np.float32)
    cov = np.stack([np.diag(v) for v in sd ** 2])
    return X, (np.full(k, 1.0 / k), means, cov)


def _oracle(Xd, r):
    """gmm_oracle.m_step on the device in fp64, and S^abs_k per component."""
    r = r.double()
    X = Xd.double()
    N = r.sum(0)
    mu = (r.T @ X) / N[:, None]
    cov, sabs = [], []
    for j in range(r.shape[1]):
        D = X - mu[j]
        cov.append(((D * r[:, j:j + 1]).T @ D / N[j]).cpu().numpy())
        A = D.abs()
        sabs.append(((A * r[:, j:j + 1]).T @ A / N[j]).cpu().numpy())
    return (N / X.shape[0]).cpu().numpy(), mu.cpu().numpy(), np.stack(cov), np.stack(sabs)


def _weighted(X, k, init, grid_limit, what):
    """One M step from init on the wgmma and the generic Gram, checked entry by entry; returns the worst ratio."""
    n, d = X.shape
    assert d > 128 or k >= 65, "the E pass must be the generic one on both paths"
    Xd = torch.from_numpy(X).cuda()
    outs = {}
    for path in (_native.PATH_AUTO, _native.PATH_GENERIC):
        with _native.Context(0) as ctx:
            ctx.set_option("kernel_path", path)
            ctx.set_option("grid_limit", grid_limit)
            ctx.reset_stats()
            outs[path] = ctx.gmm_fit(Xd, k, init=init, max_iter=1, tol=0.0)
            outs[path]["stats"] = ctx.stats()
    with _native.Context(0) as ctx:
        ctx.set_option("kernel_path", _native.PATH_GENERIC)
        r, _ = ctx.gmm_predict(Xd, *init)
    wg, gen = outs[_native.PATH_AUTO], outs[_native.PATH_GENERIC]
    assert wg["stats"]["fused_tc_launches"] >= 1, what
    assert gen["stats"]["fused_tc_launches"] == 0, what
    # the same E pass and moments pass on the same input
    assert wg["log_likelihood"] == gen["log_likelihood"], what
    assert np.array_equal(wg["weights"], gen["weights"]) and np.array_equal(wg["means"], gen["means"]), what
    w1, mu1, cov1, sabs = _oracle(Xd, r)
    np.testing.assert_allclose(gen["weights"], w1, rtol=1e-9, atol=0, err_msg=what)
    sd = np.sqrt(np.einsum("kaa->ka", sabs))
    assert (np.abs(gen["means"] - mu1) <= 1e-9 * sd).all(), what
    assert (np.abs(gen["covs"] - cov1) <= 1e-9 * sabs).all(), what
    bound = (EPS_W + 2 * n * 2.0 ** -53) * sabs
    err = np.abs(wg["covs"] - gen["covs"])
    ratio = err / np.where(bound > 0, bound, 1.0)
    worst = ratio.reshape(k, -1).max(1)
    print(f"{what}: worst |Sigma_wg - Sigma_gen| / bound = {worst.max():.3g} (component {int(worst.argmax())})")
    bad = np.argwhere(err > bound)
    assert bad.size == 0, (what, len(bad), sorted(set(int(b[0]) for b in bad))[:10],
                           [(wg["covs"][tuple(b)], gen["covs"][tuple(b)], bound[tuple(b)]) for b in bad[:3]])
    return float(worst.max())


@pytest.mark.parametrize("d,k,n,grid_limit", [
    (4, 65, 3 * RANGE + 5, 130),      # 1 tile x 65 components, P = 2 over 4 ranges
    (128, 65, 3 * RANGE + 5, 130),    # P = 2
    (132, 2, 20 * RANGE + 7, 0),      # 3 tiles x 2 components, P from the card's SM count
    (132, 2, 20 * RANGE + 7, 12),     # P = 2 over 21 ranges: 11 and 10 per CTA
    (256, 3, 3 * RANGE + 5, 18),      # 3 tiles x 3 components, P = 2
    (256, 256, 5000, 0),              # 768 CTAs: more than the SM count, P = 1
])
def test_weighted_shapes(d, k, n, grid_limit):
    X, init = _truth(n, d, k, seed=d * 1000 + k)
    _weighted(X, k, init, grid_limit, f"d={d} k={k} n={n} grid_limit={grid_limit}")


def test_weighted_separated_components():
    # D / sigma = |mu_k - mean| / sigma_k of about 11, 100 and 1100: a centre shared by all components costs component k
    # a relative error of about eps |mu_k - c|^2 / sigma_k^2 in its covariance.  The tight component is 100 times
    # tighter than the others.  Spreads are scaled by s = 0.2 at d = 132: a unit spread has a density below MLlib's EPS,
    # and a tight one below 2e-3 a density past the largest double.  Weights 5 : 1 : 5 put the mean of the mixture at
    # the origin.
    n, d, s = 3 * RANGE + 5, 132, 0.2
    rng = np.random.default_rng(3)
    u, v = np.eye(d)[0], np.eye(d)[1]
    means = s * np.stack([10 * u - 5 * v, -100 * u, 10 * u + 5 * v])
    sig = np.array([s, s, s / 100])
    w = np.array([5.0, 1.0, 5.0]) / 11
    z = rng.choice(3, size=n, p=w)
    X = (means[z] + rng.normal(size=(n, d)) * sig[z, None]).astype(np.float32)
    init = (w, means, np.stack([np.eye(d) * g ** 2 for g in sig]))
    c = X.astype(np.float64).mean(0)
    sep = np.linalg.norm(means - c, axis=1) / sig
    assert 8 < sep[0] < 15 and 80 < sep[1] < 120 and 800 < sep[2] < 1500, sep
    _weighted(X, 3, init, 18, "separated")


def test_weighted_dead_component():
    # tight rows (sigma = 0.05, d = 132) of two live components and a third one 50 units from every row: its
    # responsibilities are EPS / sum_j p_ij, 1e-116 to 1e-89, and its covariance is still a PSD one
    X, init = dead_component(3 * RANGE + 5, seed=4)
    r, _, _ = go.e_step(X[:512], *init)
    assert r[:, 2].max() < 1e-80   # fl32(r) = 0: only r / N_k keeps the weights in fp32
    _weighted(X, 3, init, 18, "dead component")
