"""PCA on the GPU: the reference's known answers through PCA(...).fit(df) / PCAModel.transform, and the device passes
(both Gram paths) against the fp64 oracle on the same float32 input."""
import json
import os

import numpy as np
import pytest

import pca_oracle as po

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")


@pytest.fixture()
def session():
    from spark_rapids_ml_b200.sparkshim import LocalSession

    return LocalSession({"spark.sql.execution.arrow.maxRecordsPerBatch": "2", "spark.rapids.ml.num_workers.local": "1"})


def _cases():
    return json.load(open(os.path.join(GOLD, "pca_known_answers.json")))


def _agree_up_to_sign(a, b, tol):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return np.allclose(a, b, atol=tol) or np.allclose(a, -b, atol=tol)


@pytest.mark.parametrize("layout", ["array", "float", "byte", "short", "int", "long"])
def test_reference_known_answers(session, tmp_path, layout):
    from spark_rapids_ml_b200.feature import PCA, PCAModel

    for name, case in _cases().items():
        data = case["data"]
        d = len(data[0])
        if layout == "array":
            df = session.createDataFrame([(r,) for r in data], ["features"])
            est = PCA(k=case["k"], num_workers=1).setInputCol("features")
        else:
            if layout != "float" and any(v != int(v) for r in data for v in r):
                continue   # integer columns: only the cases with integral data
            cols = [f"c{i}" for i in range(d)]
            ddl = ", ".join(f"{c} {layout}" for c in cols)
            df = session.createDataFrame([tuple(r) for r in data], ddl)
            est = PCA(k=case["k"], num_workers=1).setInputCol(cols)
        model = est.setOutputCol("pca").fit(df)
        ref = po.fit(np.array(data, dtype=np.float32), case["k"])
        assert model.dtype == "float32" and model.n_cols == d and model.getK() == case["k"]
        np.testing.assert_allclose(model.mean_, ref["mean_"], rtol=1e-6, atol=1e-6)
        np.testing.assert_allclose(model.components_, ref["components_"], atol=1e-5)
        np.testing.assert_allclose(model.explained_variance_ratio_, ref["explained_variance_ratio_"], atol=1e-6)
        np.testing.assert_allclose(model.singular_values_, ref["singular_values_"], rtol=1e-5, atol=1e-6)
        if "mean" in case:
            np.testing.assert_allclose(model.mean_, case["mean"], rtol=case["rel_tol"])
            assert _agree_up_to_sign(np.abs(model.components_), np.abs(case["components"]), 1e-3)
            np.testing.assert_allclose(model.explained_variance_ratio_, case["explained_variance_ratio"],
                                       rtol=case["rel_tol"])
        if "pc_columns" in case:
            np.testing.assert_allclose(model.explainedVariance, case["explained_variance_ratio"], rtol=1e-6)
            pc = np.asarray(model.pc)
            assert pc.shape == (d, case["k"])
            for j in range(case["k"]):
                assert _agree_up_to_sign(pc[:, j], case["pc_columns"][j], 1e-4)
        out = model.transform(df)
        assert out.columns[-1] == "pca"
        rows = [r["pca"] for r in out.collect()]
        Y = np.array(rows, dtype=np.float64)
        Yref = po.transform(np.array(data, dtype=np.float32), np.array(model.components_, dtype=np.float32))
        np.testing.assert_allclose(Y, Yref, atol=1e-5 * max(1.0, np.abs(Yref).max()))
        if "first_transformed_row" in case:
            for j in range(case["k"]):
                assert _agree_up_to_sign([Y[0, j]], [case["first_transformed_row"][j]], 1e-4)
        p = str(tmp_path / f"{name}_{layout}")
        model.write().overwrite().save(p)
        again = PCAModel.load(p)
        assert again.components_ == model.components_ and again.mean_ == model.mean_


def _data(kind, n, d, seed, offset=0.0):
    rng = np.random.default_rng(seed)
    if kind == "random":   # a decaying spectrum, so that most leading eigenvalues are separated
        Q, _ = np.linalg.qr(rng.normal(size=(d, d)))
        X = (rng.normal(size=(n, d)) * (1.0 / np.sqrt(1.0 + np.arange(d)))) @ Q.T + 0.1 * rng.normal(size=d)
    else:
        centers = rng.normal(scale=4.0, size=(8, d))
        X = centers[rng.integers(0, 8, size=n)] + rng.normal(size=(n, d))
    return (X + offset).astype(np.float32)


def _check_against_oracle(X, out, k, ctx):
    import torch

    n, d = X.shape
    ref = po.fit(X, k)
    lam_ref = ref["eigenvalues"][:k]
    np.testing.assert_allclose(out["mean_"], ref["mean_"], rtol=1e-6, atol=1e-6 * np.abs(ref["mean_"]).max())
    C, Cr = out["components_"], ref["components_"]
    lam = out["singular_values_"] ** 2 / (n - 1)
    if k == d:   # the covariance the device formed, reconstructed from its full eigendecomposition
        cov = C.T @ np.diag(lam) @ C
        assert np.abs(cov - ref["cov"]).max() <= 1e-5 * np.abs(ref["cov"]).max()
    gaps = po.relative_gaps(ref["eigenvalues"], k)
    checked = 0
    for i in range(k):
        if gaps[i] < 1e-3:
            continue
        assert abs(float(C[i] @ Cr[i])) >= 1 - 1e-5, (i, float(C[i] @ Cr[i]))
        top2 = np.sort(np.abs(Cr[i]))[-2:]
        if top2[1] - top2[0] > 1e-4 * top2[1]:
            assert np.sign(C[i][np.argmax(np.abs(Cr[i]))]) > 0 and float(C[i] @ Cr[i]) > 0, i
        checked += 1
    assert checked >= min(k, 3)
    assert np.abs(lam - lam_ref).max() <= 1e-5 * lam_ref[0]
    np.testing.assert_allclose(out["explained_variance_ratio_"], ref["explained_variance_ratio_"],
                               atol=1e-5 * ref["explained_variance_ratio_"][0])
    np.testing.assert_allclose(out["singular_values_"], ref["singular_values_"], atol=1e-5 * ref["singular_values_"][0])
    Xd = torch.from_numpy(X).to(ctx.device)
    Cf = C[: min(k, 32)].astype(np.float32)
    Y = ctx.pca_transform(Xd, torch.from_numpy(Cf)).cpu().numpy().astype(np.float64)
    Yr = po.transform(X, Cf)
    assert np.abs(Y - Yr).max() <= 1e-5 * np.abs(Yr).max()


@pytest.mark.parametrize("d", [20, 128, 512])
@pytest.mark.parametrize("kind", ["random", "blobs"])
@pytest.mark.parametrize("path", [0, 1])
def test_fit_matches_oracle(d, kind, path):
    import torch

    from spark_rapids_ml_b200 import _native

    n = 40000
    X = _data(kind, n, d, seed=d + (kind == "blobs"))
    with _native.Context(0) as ctx:
        ctx.set_option("kernel_path", path)
        out = ctx.pca_fit(torch.from_numpy(X).to(ctx.device), d)
        assert ctx.stats()["last_path"] == (2 if path == 0 else 1)
        _check_against_oracle(X, out, d, ctx)


@pytest.mark.parametrize("path", [0, 1])
def test_large_offset(path):
    """mean 1e3, std 1: an uncentred XᵀX - n mu muᵀ in fp32 loses every digit of the covariance."""
    import torch

    from spark_rapids_ml_b200 import _native

    X = _data("random", 1 << 20, 128, seed=11, offset=1e3)
    with _native.Context(0) as ctx:
        ctx.set_option("kernel_path", path)
        out = ctx.pca_fit(torch.from_numpy(X).to(ctx.device), 128)
        _check_against_oracle(X, out, 128, ctx)


def test_paths_agree_and_fits_are_bitwise_reproducible():
    import torch

    from spark_rapids_ml_b200 import _native

    X = _data("blobs", 70001, 256, seed=3)
    with _native.Context(0) as ctx:
        Xd = torch.from_numpy(X).to(ctx.device)
        a = ctx.pca_fit(Xd, 256)
        b = ctx.pca_fit(Xd, 256)
        for key in a:
            assert np.array_equal(a[key], b[key]), key
        ctx.set_option("kernel_path", 1)
        g = ctx.pca_fit(Xd, 256)
    np.testing.assert_allclose(a["mean_"], g["mean_"], rtol=0, atol=0)   # the same column-sum pass
    la, lg = a["singular_values_"] ** 2, g["singular_values_"] ** 2
    assert np.abs(la - lg).max() <= 1e-5 * lg[0]
    ca = a["components_"].T @ np.diag(la) @ a["components_"]
    cg = g["components_"].T @ np.diag(lg) @ g["components_"]
    assert np.abs(ca - cg).max() <= 1e-5 * np.abs(cg).max()


@pytest.mark.parametrize("d", [5, 130])
def test_unaligned_widths_take_the_generic_path(d):
    import torch

    from spark_rapids_ml_b200 import _native

    X = _data("random", 20000, d, seed=d)
    with _native.Context(0) as ctx:
        Xd = torch.from_numpy(X).to(ctx.device)
        out = ctx.pca_fit(Xd, min(d, 4))
        assert ctx.stats()["last_path"] == 1
        _check_against_oracle(X, out, min(d, 4), ctx)
        ctx.set_option("kernel_path", 2)
        with pytest.raises(_native.B2KError, match="d % 4"):
            ctx.pca_fit(Xd, 2)


def test_errors_and_zero_variance():
    import torch

    from spark_rapids_ml_b200 import _native

    with _native.Context(0) as ctx:
        X = torch.ones((100, 8), dtype=torch.float32, device=ctx.device) * 3.0
        out = ctx.pca_fit(X, 3)
        assert np.array_equal(out["components_"], np.eye(8)[:3])
        assert not out["explained_variance_ratio_"].any() and not out["singular_values_"].any()
        assert np.array_equal(out["mean_"], np.full(8, 3.0))
        with pytest.raises(_native.B2KError, match="source vector size 8 must be no less than k=9"):
            ctx.pca_fit(X, 9)
        with pytest.raises(_native.B2KError, match="k must be >= 1"):
            ctx.pca_fit(X, 0)
        with pytest.raises(_native.B2KError, match="at least 2 rows"):
            ctx.pca_fit(X[:1], 1)
        with pytest.raises(_native.B2KError, match="d <= 1024"):
            ctx.pca_fit(torch.zeros((4, 1028), dtype=torch.float32, device=ctx.device), 1)


def test_estimator_errors(session):
    from spark_rapids_ml_b200.feature import PCA

    df = session.createDataFrame([([1.0, 2.0],), ([3.0, 5.0],)], ["features"])
    with pytest.raises(Exception, match="source vector size 2 must be no less than k=3"):
        PCA(k=3, inputCol="features", num_workers=1).fit(df)
    one = session.createDataFrame([([1.0, 2.0],)], ["features"])
    with pytest.raises(Exception, match="at least 2 rows"):
        PCA(k=1, inputCol="features", num_workers=1).fit(one)


def test_transform_many_batches_one_device_pass(session):
    from spark_rapids_ml_b200.feature import PCA

    session.conf.set("spark.sql.execution.arrow.maxRecordsPerBatch", "333")
    X = _data("blobs", 5000, 48, seed=9)
    df = session.from_numpy(X, num_partitions=1)
    model = PCA(k=7, inputCol="features", outputCol="proj", num_workers=1).fit(df)
    out = model.transform(df)
    Y = np.array([r["proj"] for r in out.collect()], dtype=np.float64)
    Yr = po.transform(X, np.array(model.components_, dtype=np.float32))
    assert Y.shape == (5000, 7)
    assert np.abs(Y - Yr).max() <= 1e-5 * np.abs(Yr).max()


@pytest.mark.slow
def test_full_config4_shape_against_fp64_device_gram():
    """BASELINE config 4 per GPU: 6.25 M x 512, k = 32; covariance (k = d fit) against a chunked fp64 Gram on the device."""
    import torch

    from spark_rapids_ml_b200 import _native

    n, d = 6_250_000, 512
    g = torch.Generator(device="cuda").manual_seed(4)
    scale = (1.0 / torch.sqrt(1.0 + torch.arange(d, device="cuda", dtype=torch.float32)))
    X = torch.randn((n, d), device="cuda", generator=g) * scale + 2.0
    mu = X.sum(0, dtype=torch.float64) / n
    G = torch.zeros((d, d), dtype=torch.float64, device="cuda")
    for r in range(0, n, 1 << 18):
        xc = X[r:r + (1 << 18)].double() - mu
        G += xc.T @ xc
    cov = (G / (n - 1)).cpu().numpy()
    with _native.Context(0) as ctx:
        out = ctx.pca_fit(X, d)
        assert ctx.stats()["last_path"] == 2
        top = ctx.pca_fit(X, 32)
    np.testing.assert_allclose(out["mean_"], mu.cpu().numpy(), rtol=1e-6, atol=1e-6)
    lam = out["singular_values_"] ** 2 / (n - 1)
    covd = out["components_"].T @ np.diag(lam) @ out["components_"]
    assert np.abs(covd - cov).max() <= 1e-5 * np.abs(cov).max()
    assert np.array_equal(top["components_"], out["components_"][:32])


def _ngpu():
    import torch

    return torch.cuda.device_count()


@pytest.mark.skipif(_ngpu() < 2, reason="needs 2 GPUs")
def test_two_rank_fit_matches_single_rank():
    from spark_rapids_ml_b200.feature import PCA
    from spark_rapids_ml_b200.sparkshim import LocalSession

    s = LocalSession({"spark.sql.execution.arrow.maxRecordsPerBatch": "5000", "spark.rapids.ml.num_workers.local": "2"})
    X = _data("random", 60000, 128, seed=12)
    df = s.from_numpy(X, num_partitions=2)
    m2 = PCA(k=16, inputCol="features", num_workers=2).fit(df)
    m1 = PCA(k=16, inputCol="features", num_workers=1).fit(df)
    np.testing.assert_allclose(m2.mean_, m1.mean_, rtol=1e-6)
    np.testing.assert_allclose(m2.singular_values_, m1.singular_values_, rtol=1e-6)
    np.testing.assert_allclose(m2.explained_variance_ratio_, m1.explained_variance_ratio_, rtol=1e-6)
    for a, b in zip(m2.components_, m1.components_):
        assert abs(float(np.dot(a, b))) >= 1 - 1e-6
