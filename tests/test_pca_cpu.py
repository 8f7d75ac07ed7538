"""PCA without a GPU: the fp64 oracle against scikit-learn and the reference's known answers, the library's host eigen
step (b2k_pca_finalize) against numpy.linalg.eigh, the estimator/model params and persistence, and the pyspark-side
install proxy for pyspark.ml.feature."""
import json
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest

import pca_oracle as po
from spark_rapids_ml_b200 import _native

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
FAKE = os.path.join(ROOT, "tests", "fake_pyspark")


def _known():
    return json.load(open(os.path.join(GOLD, "pca_known_answers.json")))


def test_oracle_matches_sklearn():
    from sklearn.decomposition import PCA as SkPCA

    rng = np.random.default_rng(0)
    X = rng.normal(size=(500, 12)) @ rng.normal(size=(12, 12)) + 3.0
    ref = po.fit(X, 5)
    sk = SkPCA(n_components=5, svd_solver="full").fit(X)
    np.testing.assert_allclose(ref["mean_"], sk.mean_, rtol=1e-12)
    np.testing.assert_allclose(ref["explained_variance_ratio_"], sk.explained_variance_ratio_, rtol=1e-10)
    np.testing.assert_allclose(ref["singular_values_"], sk.singular_values_, rtol=1e-10)
    np.testing.assert_allclose(np.abs(ref["components_"]), np.abs(sk.components_), atol=1e-10)
    for a, b in zip(ref["components_"], sk.components_):
        assert abs(abs(float(a @ b)) - 1.0) < 1e-10


def test_oracle_reproduces_the_reference_known_answers():
    for name, case in _known().items():
        ref = po.fit(np.array(case["data"]), case["k"])
        if "mean" in case:
            np.testing.assert_allclose(ref["mean_"], case["mean"], rtol=case["rel_tol"])
            np.testing.assert_allclose(np.abs(ref["components_"]), np.abs(case["components"]), atol=1e-3)
            np.testing.assert_allclose(ref["explained_variance_ratio_"], case["explained_variance_ratio"],
                                       rtol=case["rel_tol"])
        if "pc_columns" in case:
            np.testing.assert_allclose(ref["explained_variance_ratio_"], case["explained_variance_ratio"], rtol=1e-9)
            for j in range(case["k"]):
                a, b = ref["components_"][j], np.array(case["pc_columns"][j])
                assert np.allclose(a, b, atol=1e-4) or np.allclose(a, -b, atol=1e-4), (name, j)
            y = po.transform(np.array(case["data"])[:1], ref["components_"])[0]
            assert np.allclose(np.abs(y), np.abs(case["first_transformed_row"]), rtol=1e-9)


def _spd(d, seed):
    rng = np.random.default_rng(seed)
    A = rng.normal(size=(d + 5, d))
    return A.T @ A / (d + 4)


@pytest.mark.parametrize("d", [2, 5, 20, 512])
def test_finalize_matches_eigh_order_and_sign(d):
    cov = _spd(d, d)
    n = 1000
    out = _native.pca_finalize(cov, n, d)
    w, V = np.linalg.eigh(cov)
    order = np.argsort(-w)
    lam = w[order]
    comp_ref = po.sign_fix(V[:, order].T)
    assert np.all(np.diff(out["singular_values_"]) <= 0)   # descending
    np.testing.assert_allclose(out["singular_values_"], np.sqrt(lam * (n - 1)), rtol=1e-10)
    np.testing.assert_allclose(out["explained_variance_ratio_"], lam / np.trace(cov), rtol=1e-9, atol=1e-15)
    gaps = po.relative_gaps(lam, d)
    for i in range(d):
        c = out["components_"][i]
        assert abs(np.linalg.norm(c) - 1) < 1e-12
        j = int(np.argmax(np.abs(c)))
        assert c[j] > 0   # sign convention
        if gaps[i] > 1e-6:
            np.testing.assert_allclose(c, comp_ref[i], atol=1e-8)


def test_finalize_repeated_eigenvalues_span_the_same_subspace():
    rng = np.random.default_rng(3)
    Q, _ = np.linalg.qr(rng.normal(size=(9, 9)))
    lam = np.array([5.0, 5.0, 5.0, 2.0, 2.0, 1.0, 0.5, 0.5, 0.1])
    cov = Q @ np.diag(lam) @ Q.T
    out = _native.pca_finalize(cov, 50, 9)
    C = out["components_"]
    np.testing.assert_allclose(C @ C.T, np.eye(9), atol=1e-12)
    np.testing.assert_allclose(out["singular_values_"] ** 2 / 49, lam, rtol=1e-12)
    for lo, hi in ((0, 3), (3, 5), (6, 8)):   # projector onto each eigenspace
        P_dev = C[lo:hi].T @ C[lo:hi]
        P_ref = Q[:, lo:hi] @ Q[:, lo:hi].T
        np.testing.assert_allclose(P_dev, P_ref, atol=1e-10)
    np.testing.assert_allclose(C.T @ np.diag(lam) @ C, cov, atol=1e-12)


def test_finalize_zero_matrix_and_errors():
    out = _native.pca_finalize(np.zeros((6, 6)), 10, 3)
    assert np.array_equal(out["components_"], np.eye(6)[:3])
    assert not out["explained_variance_ratio_"].any() and not out["singular_values_"].any()
    with pytest.raises(_native.B2KError, match="source vector size 3 must be no less than k=4"):
        _native.pca_finalize(np.eye(3), 10, 4)
    with pytest.raises(_native.B2KError, match="k must be >= 1"):
        _native.pca_finalize(np.eye(3), 10, 0)
    with pytest.raises(_native.B2KError, match="at least 2 rows"):
        _native.pca_finalize(np.eye(3), 1, 1)
    bad = np.eye(3)
    bad[0, 1] = np.nan
    with pytest.raises(_native.B2KError, match="non-finite"):
        _native.pca_finalize(bad, 10, 1)


def test_params_defaults_aliases_and_copy():
    from spark_rapids_ml_b200.feature import PCA

    p = PCA()
    assert p.cuml_params == {"n_components": None, "svd_solver": "auto", "verbose": False, "whiten": False}
    assert not p.isDefined("k") and p.getOutputCol() == p.uid + "__output"
    with pytest.raises(ValueError, match="k is not set"):
        p._validate_parameters()
    p = PCA(k=3, inputCol="f", outputCol="o", svd_solver="full", whiten=True)
    assert p.getK() == 3 and p.cuml_params["n_components"] == 3 and p.getInputCol() == "f" and p.getOutputCol() == "o"
    assert p.cuml_params["svd_solver"] == "full" and p.cuml_params["whiten"] is True
    with pytest.raises(ValueError, match="set one or the other"):
        PCA(k=2, n_components=3)
    assert PCA(n_components=4).getK() == 4
    with pytest.raises(ValueError, match="must be > 0"):
        PCA(k=0)._validate_parameters()
    q = PCA(inputCol=["a", "b"])
    assert q.getInputCol() == ["a", "b"] and q._get_input_columns() == (None, ["a", "b"])
    assert PCA().setInputCol("x")._get_input_columns() == ("x", None)
    assert PCA().setInputCols(["x", "y"]).getInputCols() == ["x", "y"]
    c = p.copy({p.k: 5})
    assert c.getK() == 5 and c.cuml_params["n_components"] == 5 and p.getK() == 3


def test_model_surface_and_persistence(tmp_path):
    from spark_rapids_ml_b200.feature import PCA, PCAModel

    est = PCA(k=2, inputCol="feats", outputCol="proj")
    est.save(str(tmp_path / "est"))
    e2 = PCA.load(str(tmp_path / "est"))
    assert e2.uid == est.uid and e2.getK() == 2 and e2.getInputCol() == "feats" and e2.getOutputCol() == "proj"
    assert e2.cuml_params["n_components"] == 2
    m = PCAModel(mean_=[1.0, 2.0, 3.0], components_=[[1.0, 0.0, 0.0], [0.0, 0.6, 0.8]],
                 explained_variance_ratio_=[0.7, 0.2], singular_values_=[3.0, 1.5], n_cols=3, dtype="float32")
    est._copyValues(m)
    assert m.getK() == 2 and m.cuml_params["n_components"] == 2 and m.mean == [1.0, 2.0, 3.0]
    assert np.array_equal(m.pc, np.array([[1.0, 0.0], [0.0, 0.6], [0.0, 0.8]]))
    assert np.array_equal(m.explainedVariance, np.array([0.7, 0.2]))
    assert m._output_col_name() == "proj" and m._out_schema(None) == "array<float>"
    with pytest.raises(NotImplementedError):
        m.cpu()
    m.write().overwrite().save(str(tmp_path / "model"))
    m2 = PCAModel.load(str(tmp_path / "model"))
    assert m2.uid == m.uid and m2.components_ == m.components_ and m2.mean_ == m.mean_ and m2.getOutputCol() == "proj"
    assert m2.singular_values_ == m.singular_values_ and m2.explained_variance_ratio_ == m.explained_variance_ratio_


def test_directory_written_by_the_reference_loads_here(tmp_path):
    """The reference's _CumlModelWriter layout: metadata/part-00000 (DefaultParamsWriter JSON + the cuML params) and
    data/part-00000 = json.dumps(model attributes), with Hadoop _SUCCESS markers."""
    from spark_rapids_ml_b200.feature import PCAModel

    path = tmp_path / "ref_pca_model"
    meta = {"class": "spark_rapids_ml.feature.PCAModel", "timestamp": 1700000000000, "sparkVersion": "3.5.1",
            "uid": "PCA_5b8e2d9c1a07", "paramMap": {"k": 2, "inputCol": "features", "outputCol": "pca_features"},
            "defaultParamMap": {"outputCol": "PCA_5b8e2d9c1a07__output"},
            "_cuml_params": {"n_components": 2, "svd_solver": "auto", "verbose": False, "whiten": False},
            "_num_workers": 2, "_float32_inputs": True}
    attrs = {"mean_": [3.0, 2.0], "components_": [[1.0, 0.0], [0.0, 1.0]], "explained_variance_ratio_": [0.8, 0.2],
             "singular_values_": [4.0, 2.0], "n_cols": 2, "dtype": "float32"}
    for sub, obj in (("metadata", meta), ("data", attrs)):
        os.makedirs(path / sub)
        (path / sub / "part-00000").write_text(json.dumps(obj) + "\n")
        (path / sub / "_SUCCESS").write_text("")
    m = PCAModel.load(str(path))
    assert m.uid == "PCA_5b8e2d9c1a07" and m.getK() == 2 and m.getInputCol() == "features"
    assert m.getOutputCol() == "pca_features" and m._num_workers == 2 and m.n_cols == 2
    assert m.components_ == [[1.0, 0.0], [0.0, 1.0]] and m.mean_ == [3.0, 2.0]


_FAKE_PYSPARK = '''
import sys, json
import pyspark.ml.feature as stock_mod
StockPCA = stock_mod.PCA
import spark_rapids_ml_b200.sparkshim as shim
assert shim.HAVE_PYSPARK
import spark_rapids_ml_b200.install as inst
from spark_rapids_ml_b200.feature import PCA, PCAModel
from pyspark.ml.feature import PCA as P1, PCAModel as M1, StandardScaler as S1
import pyspark.ml, pyspark.ml.param
res = {
    "user_import_is_accelerated": P1 is PCA and M1 is PCAModel and pyspark.ml.feature.PCA is PCA,
    "other_names_untouched": getattr(S1, "stock", False) is True,
    "estimator_and_model_types": issubclass(PCA, pyspark.ml.Estimator) and issubclass(PCAModel, pyspark.ml.Model),
    "pyspark_params": isinstance(PCA().getParam("k"), pyspark.ml.param.Param),
}
p = PCA(k=2, inputCol="f", outputCol="o")
res["params"] = [p.getK(), p.getInputCol(), p.getOutputCol(), p.cuml_params["n_components"]]
inst.uninstall()
res["uninstall_restores"] = sys.modules["pyspark.ml.feature"].PCA is StockPCA
print("RESULT " + json.dumps(res))
'''


def test_install_proxy_and_pyspark_params_for_feature_pca():
    env = dict(os.environ)
    env["PYTHONPATH"] = os.pathsep.join([FAKE, ROOT, env.get("PYTHONPATH", "")])
    r = subprocess.run([sys.executable, "-c", textwrap.dedent(_FAKE_PYSPARK)], env=env, capture_output=True, text=True,
                       timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    res = json.loads([ln for ln in r.stdout.splitlines() if ln.startswith("RESULT ")][-1][len("RESULT "):])
    for key in ("user_import_is_accelerated", "other_names_untouched", "estimator_and_model_types", "pyspark_params",
                "uninstall_restores"):
        assert res[key] is True, (key, res)
    assert res["params"] == [2, "f", "o", 2], res
