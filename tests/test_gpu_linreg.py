"""Linear regression on the GPU: the moments pass on both Gram paths against an fp64 restatement on the device, fits
through the estimator against the fp64 oracle in the solver's frame, MLlib's known answers end to end, determinism, the
single-pass fitMultiple, transform, and errors.

Tolerances.  The wgmma Gram pass forms products in 3xTF32 with fp64 partials every 4096 rows; PCA measured 2.7e-7
max|G| at 6.25 M x 512, and 4e-6 max|G| bounds it with margin for the shapes here.  The generic Gram pass (PCA's, shared
unchanged) centres each value in fp32, which rounds it by at most 2^-24 relative, then multiplies and sums in fp64: an
entry is within (2^-23 + n 2^-53) sum |v_i v_j| of the exact one, and that elementwise bound is what the moments test
holds it to.  k_xty centres, multiplies and sums in fp64, so X^T y and y^T y are held to 1e-10 of their Cauchy-Schwarz
scale on both paths.  In the solver's frame (A = Z^T Z / n + l2 I, c = Z^T t / n) an entry of A is then off by at most
eps max|A|, with eps = 4e-6 on wgmma and, by Cauchy-Schwarz on the bound above, 2^-22 on the generic path; c is exact
to 1e-10.  That moves the residual of the device's solution v against the exact system by at most
eps (max|A| |v|_1 + max|c|): the backward-error rule the closed forms meet, and the slack granted to the KKT
conditions of coordinate descent run to tol = 1e-12.
"""
import json
import os

import numpy as np
import pytest

import linreg_oracle as lo

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EPS = {2: 4e-6, 1: 2.0 ** -22}   # last_path -> the bound on an entry error of A relative to max|A| (see above)


@pytest.fixture(scope="module")
def session():
    from spark_rapids_ml_b200.sparkshim import LocalSession

    return LocalSession({"spark.sql.execution.arrow.maxRecordsPerBatch": "1000", "spark.rapids.ml.num_workers.local": "1"})


def _data(n, d, seed, offset=0.0):
    rng = np.random.default_rng(seed)
    X = (rng.normal(size=(n, d)) + offset).astype(np.float32)
    w = rng.normal(size=d)
    y = ((X.astype(np.float64) - offset) @ w + 1.5 + offset + 0.3 * rng.normal(size=n)).astype(np.float32)
    return X, y


def _device_moments(Xd, yd):
    """fp64 means, centred moments and sum |v_i v_j| of [X | y], on the device."""
    import torch

    V = torch.cat([Xd.double(), yd.double()[:, None]], 1)
    m = V.mean(0)
    C = V - m
    return m.cpu().numpy(), (C.T @ C).cpu().numpy(), (C.abs().T @ C.abs()).cpu().numpy()


def _check_moments(ctx, X, y, path):
    import torch

    Xd, yd = torch.from_numpy(X).cuda(), torch.from_numpy(y).cuda()
    ctx.set_option("kernel_path", path)
    n, mean, M = ctx.linreg_moments(Xd, yd)
    last = ctx.stats()["last_path"]
    ctx.set_option("kernel_path", 0)
    m_ref, M_ref, S = _device_moments(Xd, yd)
    d = X.shape[1]
    assert n == X.shape[0]
    np.testing.assert_allclose(mean, m_ref, rtol=1e-12, atol=1e-12 * np.abs(m_ref).max())
    G, G_ref = M[:d, :d], M_ref[:d, :d]
    if last == 2:
        assert np.abs(G - G_ref).max() <= EPS[last] * np.abs(G_ref).max(), (d, last)
    else:
        assert (np.abs(G - G_ref) <= (2.0 ** -23 + n * 2.0 ** -53) * S[:d, :d]).all(), (d, last)
    cs = np.sqrt(np.outer(np.diag(M_ref), np.diag(M_ref)))[d]   # Cauchy-Schwarz scale of row d (the label)
    assert (np.abs(M[d] - M_ref[d]) <= 1e-10 * cs).all(), (d, last)
    assert np.array_equal(M, M.T)
    return last


@pytest.mark.parametrize("d", [1, 3, 5, 20, 128, 512, 1024])
def test_moments_on_both_paths(d):
    from spark_rapids_ml_b200 import _native

    X, y = _data(20000 if d < 1024 else 6000, d, d)
    with _native.Context(0) as ctx:
        paths = [_check_moments(ctx, X, y, 1)]
        if d % 4 == 0:
            paths.append(_check_moments(ctx, X, y, 2))
            paths.append(_check_moments(ctx, X, y, 0))
    assert paths == ([1, 2, 2] if d % 4 == 0 else [1])


@pytest.mark.parametrize("path", [1, 2])
def test_large_offset(path):
    from spark_rapids_ml_b200 import _native

    X, y = _data(50000, 64, 11, offset=1e3)
    with _native.Context(0) as ctx:
        assert _check_moments(ctx, X, y, path) == path


def _fit(session, X, y, **kw):
    from spark_rapids_ml_b200.regression import LinearRegression

    df = session.from_numpy(X, num_partitions=1, extra={"label": y})
    return LinearRegression(num_workers=1, **kw).fit(df)


@pytest.mark.parametrize("path", [1, 2])
@pytest.mark.parametrize("fi", [True, False])
@pytest.mark.parametrize("st", [True, False])
@pytest.mark.parametrize("reg,l1", [(0.0, 0.0), (0.3, 0.0), (0.05, 1.0), (0.05, 0.5)])
def test_fits_against_the_oracle(session, monkeypatch, path, fi, st, reg, l1):
    from spark_rapids_ml_b200 import _native

    orig = _native.Context.__init__

    def with_path(self, *a, **k):
        orig(self, *a, **k)
        self.set_option("kernel_path", path)

    monkeypatch.setattr(_native.Context, "__init__", with_path)
    X, y = _data(30000, 32, 21, offset=2.0)
    model = _fit(session, X, y, regParam=reg, elasticNetParam=l1, fitIntercept=fi, standardization=st,
                 tol=1e-12, maxIter=100000)
    f = lo.frame(X, y, fi, st)
    lam = reg / f["sy"]
    l1w, l2w = lam * l1, lam * (1 - l1)
    A = f["A"] + l2w * np.eye(32)
    c = f["c"]
    v = lo.solver_frame_v(np.asarray(model.coef_), f)
    slack = EPS[path] * (np.abs(A).max() * np.abs(v).sum() + np.abs(c).max())
    if reg == 0.0 or l1 == 0.0:
        assert np.abs(A @ v - c).max() <= slack
    else:
        assert lo.kkt_residual(f["A"], c, v, l1w, l2w) <= slack
    if fi:
        assert model.intercept == pytest.approx(f["muy"] - np.asarray(model.coef_) @ f["mu"], rel=1e-12, abs=1e-12)
    else:
        assert model.intercept == 0.0


def test_mllib_known_answers_end_to_end(session):
    k = json.load(open(os.path.join(ROOT, "tests", "golden", "linreg_known_answers.json")))
    X, y = np.array(k["X"], dtype=np.float32), np.array(k["y"], dtype=np.float32)
    for name, c in k["cases"].items():
        m = _fit(session, X, y, regParam=c["regParam"], elasticNetParam=c["elasticNetParam"], maxIter=200)
        np.testing.assert_allclose(np.asarray(m.coefficients), c["coefficients"], rtol=1e-6, err_msg=name)
        # intercept = muy - w.mu: a coefficient error of 1e-6 relative moves it by 1e-6 (|muy| + sum |w_j mu_j|)
        scale = abs(float(y.astype(np.float64).mean())) + float(np.abs(np.asarray(m.coef_) * X.mean(0, dtype=np.float64)).sum())
        assert abs(m.intercept - c["intercept"]) <= c.get("intercept_atol", 1e-6 * scale), name
        if "first_prediction" in c:
            df = session.from_numpy(X, num_partitions=1, extra={"label": y})
            pred = m.transform(df).collect()[0]["prediction"]
            assert pred == pytest.approx(c["first_prediction"], rel=1e-6)


def test_two_fits_are_bitwise_equal(session):
    X, y = _data(40000, 128, 31)
    a = _fit(session, X, y, regParam=0.1, elasticNetParam=0.5)
    b = _fit(session, X, y, regParam=0.1, elasticNetParam=0.5)
    assert a.coef_ == b.coef_ and a.intercept_ == b.intercept_


def test_fit_multiple_is_one_pass(session, monkeypatch):
    from spark_rapids_ml_b200 import _native
    from spark_rapids_ml_b200.regression import LinearRegression

    launches = []
    orig = _native.Context.linreg_moments

    def counted(self, X, y):
        out = orig(self, X, y)
        launches.append(self.stats()["kernel_launches"])
        return out

    monkeypatch.setattr(_native.Context, "linreg_moments", counted)
    X, y = _data(30000, 64, 41)
    df = session.from_numpy(X, num_partitions=1, extra={"label": y})
    lr = LinearRegression(num_workers=1)
    maps = [{lr.regParam: r, lr.elasticNetParam: a} for r in (0.0, 0.2) for a in (0.0, 0.5, 1.0)]
    models = dict(lr.fitMultiple(df, maps))
    assert len(launches) == 1
    singles = [lr.copy(pm).fit(df) for pm in maps]
    assert len(launches) == 7 and all(n == launches[0] for n in launches)
    for i, s in enumerate(singles):
        assert models[i].coef_ == s.coef_ and models[i].intercept_ == s.intercept_
        assert models[i].getRegParam() == s.getRegParam() and models[i].getElasticNetParam() == s.getElasticNetParam()


@pytest.mark.parametrize("d", [1, 7, 128])
def test_transform_many_batches_one_device_pass(session, d):
    X, y = _data(5000, d, 51)
    model = _fit(session, X, y, regParam=0.01)
    session.conf.set("spark.sql.execution.arrow.maxRecordsPerBatch", "333")
    try:
        df = session.from_numpy(X, num_partitions=2, extra={"label": y})
        out = model.transform(df)
    finally:
        session.conf.set("spark.sql.execution.arrow.maxRecordsPerBatch", "1000")
    pred = np.array([r["prediction"] for r in out.collect()], dtype=np.float64)
    assert str(dict(out.dtypes)["prediction"]) == "double"
    terms = X.astype(np.float64) * np.asarray(model.coef_)
    ref = model.intercept + terms.sum(1)
    bound = d * 2.0 ** -52 * (np.abs(terms).sum(1) + abs(model.intercept))
    assert (np.abs(pred - ref) <= bound).all()
    empty = session.from_numpy(X[:0], num_partitions=1, extra={"label": y[:0]})
    assert model.transform(empty).count() == 0
    wrong = session.from_numpy(np.zeros((10, d + 1), np.float32), num_partitions=1)
    with pytest.raises(Exception):
        model.transform(wrong).collect()


def test_predict_paths_give_the_same_bits():
    """The float4 and scalar loads read the same features in the same order: an unaligned X gives the same bits."""
    import torch

    from spark_rapids_ml_b200 import _native

    X, _ = _data(10001, 64, 61)
    w = np.random.default_rng(0).normal(size=64)
    with _native.Context(0) as ctx:
        buf = torch.from_numpy(np.concatenate([np.zeros(1, np.float32), X.reshape(-1)])).cuda()
        aligned = torch.from_numpy(X).cuda()
        a = ctx.linreg_predict(aligned, w, 0.5).cpu().numpy()
        b = ctx.linreg_predict(buf[1:].view(10001, 64), w, 0.5).cpu().numpy()
    assert np.array_equal(a, b)


def test_non_finite_rows_and_errors(session):
    import torch

    from spark_rapids_ml_b200 import _native

    X, y = _data(2000, 8, 71)
    with _native.Context(0) as ctx:
        for bad in ("x_nan", "x_inf", "y_nan"):
            Xb, yb = X.copy(), y.copy()
            if bad == "x_nan":
                Xb[17, 3] = np.nan
            elif bad == "x_inf":
                Xb[5, 0] = np.inf
            else:
                yb[100] = np.nan
            with pytest.raises(_native.B2KError, match="NaN or an infinity"):
                ctx.linreg_moments(torch.from_numpy(Xb).cuda(), torch.from_numpy(yb).cuda())
        with pytest.raises(_native.B2KError, match="d <= 1024"):
            ctx.linreg_moments(torch.zeros((4, 1025), device="cuda"), torch.zeros(4, device="cuda"))
    Xb = X.copy()
    Xb[0, 0] = np.nan
    with pytest.raises(Exception, match="NaN or an infinity"):
        _fit(session, Xb, y)


def _ngpu():
    import torch

    return torch.cuda.device_count()


@pytest.mark.skipif(_ngpu() < 2, reason="needs 2 GPUs")
def test_two_rank_fit_matches_single_rank():
    from spark_rapids_ml_b200.regression import LinearRegression
    from spark_rapids_ml_b200.sparkshim import LocalSession

    s = LocalSession({"spark.sql.execution.arrow.maxRecordsPerBatch": "5000", "spark.rapids.ml.num_workers.local": "2"})
    X, y = _data(60000, 128, 81)
    df = s.from_numpy(X, num_partitions=2, extra={"label": y})
    m2 = LinearRegression(num_workers=2, regParam=0.1).fit(df)
    m1 = LinearRegression(num_workers=1, regParam=0.1).fit(df)
    np.testing.assert_allclose(m2.coef_, m1.coef_, rtol=1e-6, atol=1e-9)
    assert m2.intercept == pytest.approx(m1.intercept, rel=1e-6)
