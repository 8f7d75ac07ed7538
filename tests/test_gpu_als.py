"""b2k_als_fit / _predict / _recommend on the device against the fp64 oracle of tests/als_oracle.py: one iteration from
injected factors (explicit and implicit) within the oracle's per-system bound, a full fit's factors and RMSE, the edges
(ranks 1 to 128 and 129, a single-rating user, a destination of many units, power-law degrees, duplicate pairs,
negative implicit ratings, ids at +-(2^31 - 1), a system that is not positive definite, a NaN rating), a capped grid,
bitwise repeats, predictions bitwise equal to NumPy's float32 rank-order dot, and top-n recommendations bitwise equal
to the oracle's from the same scores."""
import numpy as np
import pytest

import als_oracle as ao

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    from spark_rapids_ml_b200 import _native

    with _native.Context(0) as c:
        yield c


def _t(a, dtype):
    import torch

    return torch.from_numpy(np.ascontiguousarray(a, dtype=dtype)).cuda()


def ratings(n_users, n_items, n, seed, power=False, implicit=False):
    rng = np.random.default_rng(seed)
    if power:   # Zipf-like degrees on both sides
        u = np.minimum((rng.pareto(1.2, n) * n_users / 20).astype(np.int64), n_users - 1)
        i = np.minimum((rng.pareto(1.2, n) * n_items / 20).astype(np.int64), n_items - 1)
    else:
        u = rng.integers(0, n_users, n)
        i = rng.integers(0, n_items, n)
    u = u * 7 - 1000   # raw ids: sparse, some negative
    i = i * 3 + 5
    r = rng.normal(size=n) * 2 if implicit else rng.integers(1, 6, n).astype(np.float64)
    return u.astype(np.float64), i.astype(np.float64), r.astype(np.float32)


def run(ctx, u, i, r, rank, **kw):
    out = ctx.als_fit(_t(u, np.float64), _t(i, np.float64), None if r is None else _t(r, np.float32), rank=rank, **kw)
    return {k: v.cpu().numpy() for k, v in out.items()}


def check_one_iteration(ctx, u, i, r, rank, reg, implicit=False, alpha=1.0):
    uid, iid, du, di = ao.index(u, i)
    U0 = ao.start(uid, rank, 11)
    out = run(ctx, u, i, r, rank, max_iter=1, reg_param=reg, implicit_prefs=implicit, alpha=alpha, init_user_factors=U0)
    np.testing.assert_array_equal(out["user_ids"], uid)
    np.testing.assert_array_equal(out["item_ids"], iid)
    IF, ci = ao.half_step(di, du, r, U0, len(iid), reg, implicit, alpha)
    assert np.all(np.abs(out["item_factors"] - IF) <= ao.step_tol(IF, ci)), np.abs(out["item_factors"] - IF).max()
    UF, cu = ao.half_step(du, di, r, out["item_factors"], len(uid), reg, implicit, alpha)
    assert np.all(np.abs(out["user_factors"] - UF) <= ao.step_tol(UF, cu)), np.abs(out["user_factors"] - UF).max()
    return out


@pytest.mark.parametrize("rank", [1, 4, 10, 64, 128])
@pytest.mark.parametrize("implicit", [False, True])
def test_one_iteration_matches_oracle(ctx, rank, implicit):
    u, i, r = ratings(300, 200, 6000, seed=rank, implicit=implicit)
    check_one_iteration(ctx, u, i, r, rank, 0.1, implicit, alpha=2.0)


def test_rank_129_unsupported(ctx):
    from spark_rapids_ml_b200._native import B2KError

    u, i, r = ratings(30, 20, 200, seed=0)
    with pytest.raises(B2KError, match="rank <= 128") as e:
        run(ctx, u, i, r, 129)
    assert e.value.code == 4


def test_edges_single_rating_long_destination_power_law_duplicates(ctx):
    u, i, r = ratings(500, 300, 20000, seed=3, power=True)
    # one user with a single rating, one item rated 3000 times (six units), and duplicated pairs
    u = np.concatenate([u, [123457.0], np.full(3000, 5.0), u[:500]])
    i = np.concatenate([i, [8.0], np.full(3000, 999999.0), i[:500]])
    r = np.concatenate([r, [4.0], (np.arange(3000) % 5 + 1).astype(np.float32), r[:500] + 1]).astype(np.float32)
    check_one_iteration(ctx, u, i, r, 10, 0.05)
    check_one_iteration(ctx, u, i, r, 10, 0.05, implicit=True)


def test_negative_implicit_ratings_and_extreme_ids(ctx):
    u, i, r = ratings(100, 80, 3000, seed=4, implicit=True)
    u[:40] = 2.0 ** 31 - 1
    u[40:80] = -(2.0 ** 31 - 1)
    i[:20] = -(2.0 ** 31)
    out = check_one_iteration(ctx, u, i, r, 8, 0.1, implicit=True, alpha=0.5)
    assert out["user_ids"][0] == -(2 ** 31 - 1) and out["user_ids"][-1] == 2 ** 31 - 1
    assert out["item_ids"][0] == -(2 ** 31)


def test_full_fit_and_rmse(ctx):
    rng = np.random.default_rng(5)
    P, Qm = rng.normal(size=(200, 4)), rng.normal(size=(150, 4))
    n = 8000
    uu, ii = rng.integers(0, 200, n), rng.integers(0, 150, n)
    r = (np.einsum("ij,ij->i", P[uu], Qm[ii]) + 0.1 * rng.normal(size=n)).astype(np.float32)
    u, i = uu.astype(np.float64), ii.astype(np.float64)
    out = run(ctx, u, i, r, 4, max_iter=10, reg_param=0.01, seed=3)
    ref = ao.fit(u, i, r, 4, 10, 0.01, seed=3)
    np.testing.assert_allclose(out["user_factors"], ref["user_factors"], rtol=1e-3, atol=1e-4)
    np.testing.assert_allclose(out["item_factors"], ref["item_factors"], rtol=1e-3, atol=1e-4)
    _, _, du, di = ao.index(u, i)
    pred = ao.predict(out["user_factors"][du], out["item_factors"][di])
    pref = ao.predict(ref["user_factors"][du], ref["item_factors"][di])
    rmse = np.sqrt(np.mean((pred - r) ** 2))
    assert abs(rmse - np.sqrt(np.mean((pref - r) ** 2))) <= 1e-4 and rmse < 0.2, rmse


def test_seeded_start_matches_oracle(ctx):
    u, i, r = ratings(300, 100, 3000, seed=6)
    out = run(ctx, u, i, r, 16, max_iter=0, seed=42)
    np.testing.assert_allclose(out["user_factors"], ao.start(out["user_ids"], 16, 42), rtol=1e-6, atol=1e-7)


def test_not_positive_definite_and_nan_rating_fail(ctx):
    from spark_rapids_ml_b200._native import B2KError

    u, i, r = ratings(50, 40, 600, seed=7)
    # start factors with a zero last coordinate: every item's A has an exactly zero row, and regParam = 0 adds nothing
    U0 = ao.start(ao.index(u, i)[0], 4, 1)
    U0[:, -1] = 0.0
    with pytest.raises(B2KError, match="not positive definite"):
        run(ctx, u, i, r, 4, max_iter=1, reg_param=0.0, init_user_factors=U0)
    r2 = r.copy()
    r2[17] = np.nan
    with pytest.raises(B2KError, match="finite ratings"):
        run(ctx, u, i, r2, 4)
    u2 = u.copy()
    u2[3] = 1.5
    with pytest.raises(B2KError, match="column user. Value 1.5 was either"):
        run(ctx, u2, i, r, 4)


def test_capped_grid_and_repeats_are_bitwise_equal(ctx):
    u, i, r = ratings(800, 500, 60000, seed=8, power=True)
    a = run(ctx, u, i, r, 32, max_iter=2, seed=1)
    b = run(ctx, u, i, r, 32, max_iter=2, seed=1)
    ctx.set_option("grid_limit", 3)
    try:
        c = run(ctx, u, i, r, 32, max_iter=2, seed=1)
    finally:
        ctx.set_option("grid_limit", 0)
    for k in a:
        np.testing.assert_array_equal(a[k], b[k])
        np.testing.assert_array_equal(a[k], c[k])


def test_predict_and_recommend_bitwise(ctx):
    import torch

    u, i, r = ratings(300, 250, 8000, seed=9)
    out = ctx.als_fit(_t(u, np.float64), _t(i, np.float64), _t(r, np.float32), rank=12, max_iter=3, seed=2)
    UF, IF = out["user_factors"].cpu().numpy(), out["item_factors"].cpu().numpy()
    uid, iid = out["user_ids"].cpu().numpy(), out["item_ids"].cpu().numpy()
    qu = np.concatenate([u[:500], [1e9, 2.5]])
    qi = np.concatenate([i[:500], [i[0], i[1]]])
    p = ctx.als_predict(_t(qu, np.float64), _t(qi, np.float64), out["user_ids"], out["user_factors"],
                        out["item_ids"], out["item_factors"]).cpu().numpy()
    ref = ao.predict(UF[np.searchsorted(uid, qu[:500])], IF[np.searchsorted(iid, qi[:500])])
    np.testing.assert_array_equal(p[:500].view(np.int32), ref.view(np.int32))
    assert np.isnan(p[500:]).all()
    # ties: duplicate target rows score equal; the lower row must come first
    T = np.concatenate([IF, IF[:40]]).astype(np.float32)
    for n in (1, 7, 300, 1024):
        idx, sc = ctx.als_recommend(out["user_factors"], torch.from_numpy(T).cuda(), n)
        ridx, rsc = ao.recommend(UF, T, n)
        k = ridx.shape[1]
        np.testing.assert_array_equal(idx.cpu().numpy()[:, :k], ridx)
        np.testing.assert_array_equal(sc.cpu().numpy()[:, :k].view(np.int32), rsc.view(np.int32))
        assert (idx.cpu().numpy()[:, k:] == -1).all()
