"""GaussianMixture without a GPU: the fp64 oracle (densities against scipy, the pseudo-inverse of a singular
covariance, the start's independence from partitioning, a log-likelihood that never decreases) and the estimator /
model surface (params, defaults, validation, copy, persistence)."""
import numpy as np
import pytest
from scipy.stats import multivariate_normal

import gmm_oracle as go
from spark_rapids_ml_b200.clustering import GaussianMixture, GaussianMixtureModel


def _mixture(n, d, k, seed, shift=0.0):
    rng = np.random.default_rng(seed)
    means = rng.normal(scale=6.0, size=(k, d))
    z = rng.integers(0, k, size=n)
    A = rng.normal(size=(k, d, d)) / np.sqrt(d)
    X = means[z] + np.einsum("nij,nj->ni", A[z], rng.normal(size=(n, d))) + shift
    return X.astype(np.float32)


def test_density_matches_scipy_for_full_rank_covariances():
    rng = np.random.default_rng(1)
    for d in (1, 3, 8):
        A = rng.normal(size=(d, d))
        cov = A @ A.T + 0.5 * np.eye(d)
        mu = rng.normal(size=d)
        X = rng.normal(size=(50, d)) * 2
        np.testing.assert_allclose(go.log_pdf(X, mu, cov), multivariate_normal(mu, cov).logpdf(X), rtol=1e-10,
                                   atol=1e-10)


def test_pseudo_inverse_on_a_rank_deficient_covariance():
    # rank 2 in 3 dimensions: the density lives on the plane and uses the pseudo-determinant
    rng = np.random.default_rng(2)
    B = rng.normal(size=(3, 2))
    cov = B @ B.T
    mu = rng.normal(size=3)
    X = mu + rng.normal(size=(20, 2)) @ B.T
    lam, U = np.linalg.eigh(cov)
    keep = lam > go.EPS * lam.max() * 3
    assert keep.sum() == 2
    pinv = (U[:, keep] / lam[keep]) @ U[:, keep].T
    q = np.einsum("ni,ij,nj->n", X - mu, pinv, X - mu)
    want = -0.5 * (3 * np.log(2 * np.pi) + np.log(lam[keep]).sum()) - 0.5 * q
    np.testing.assert_allclose(go.log_pdf(X, mu, cov), want, rtol=1e-9)
    with pytest.raises(ValueError, match="no eigenvalue"):
        go.log_pdf(X, mu, np.zeros((3, 3)))


def test_init_rule_does_not_depend_on_partitioning():
    X = _mixture(300, 4, 3, 3)
    rows = go.init_rows(7, 3, 300)
    assert rows.shape == (15,) and rows.min() >= 0 and rows.max() < 300
    w, mu, cov = go.random_init(X, 3, 7)
    # the rule reads global rows only: any split of X into consecutive rank shards gives the same rows
    for cuts in ([100], [1, 299], [50, 120, 260]):
        shards = np.split(X, cuts)
        Xg = np.concatenate(shards)
        w2, mu2, cov2 = go.random_init(Xg, 3, 7)
        np.testing.assert_array_equal(mu, mu2)
        np.testing.assert_array_equal(cov, cov2)
    np.testing.assert_array_equal(w, np.full(3, 1 / 3))
    assert np.all(cov[:, np.arange(4), np.arange(4)] >= 0)
    assert not np.array_equal(go.init_rows(8, 3, 300), rows)


def test_log_likelihood_never_decreases():
    X = _mixture(600, 3, 4, 4, shift=100.0)
    w, mu, cov = go.random_init(X, 4, 11)
    _, _, _, ll, it, hist = go.fit(X, w, mu, cov, 40, 0.0)
    assert it >= 5
    assert all(b >= a - 1e-7 * abs(a) for a, b in zip(hist, hist[1:])), hist


def test_e_step_rows_sum_to_one_and_ties_go_low():
    X = np.zeros((2, 2))
    w = np.array([0.5, 0.5])
    mu = np.zeros((2, 2))
    cov = np.stack([np.eye(2), np.eye(2)])
    r, _, lab = go.e_step(X, w, mu, cov)
    np.testing.assert_allclose(r.sum(axis=1), 1.0)
    assert list(lab) == [0, 0]


def test_params_defaults_and_setters():
    est = GaussianMixture()
    assert est.getK() == 2 and est.getMaxIter() == 100 and est.getTol() == 0.01
    assert est.getProbabilityCol() == "probability" and est.getPredictionCol() == "prediction"
    assert est.getFeaturesCol() == "features" and est.getAggregationDepth() == 2
    assert est.getSeed() == hash("GaussianMixture") & 0x07FFFFFFF
    est = GaussianMixture(k=5, maxIter=7, tol=0.5, seed=3, probabilityCol="p", featuresCol=["a", "b"])
    assert est.cuml_params["n_components"] == 5 and est.cuml_params["max_iter"] == 7
    assert est.cuml_params["tol"] == 0.5 and est.cuml_params["random_state"] == 3
    assert est.getFeaturesCol() == ["a", "b"] and est.getProbabilityCol() == "p"
    est.setK(4).setMaxIter(3).setTol(0.0).setSeed(9).setAggregationDepth(3)
    assert (est.getK(), est.getMaxIter(), est.getTol(), est.getSeed()) == (4, 3, 0.0, 9)
    c = est.copy({est.k: 6})
    assert c.getK() == 6 and c.cuml_params["n_components"] == 6 and est.getK() == 4


@pytest.mark.parametrize("kw,msg", [({"k": 1}, "k given invalid"), ({"maxIter": -1}, "maxIter given invalid"),
                                    ({"tol": -0.5}, "tol given invalid")])
def test_validation_errors(kw, msg):
    with pytest.raises(ValueError, match=msg):
        GaussianMixture(**kw)._validate_parameters()


def test_weight_col_raises():
    with pytest.raises(ValueError, match="weightCol"):
        GaussianMixture(weightCol="w")
    with pytest.raises(ValueError, match="weightCol"):
        GaussianMixture().setWeightCol("w")


def _model():
    return GaussianMixtureModel(weights_=[0.25, 0.75], means_=[[0.0, 1.0], [2.0, 3.0]],
                                covs_=[[[1.0, 0.1], [0.1, 2.0]], [[0.5, 0.0], [0.0, 0.5]]], cluster_sizes_=[3, 9],
                                log_likelihood_=-12.5, num_iters=4, n_cols=2, dtype="float32")


def test_model_surface_and_persistence(tmp_path):
    m = _model()
    m.setProbabilityCol("prob")
    assert m.weights == [0.25, 0.75] and m.hasSummary and m.getK() == 2
    s = m.summary
    assert (s.k, s.numIter, s.logLikelihood, s.clusterSizes) == (2, 4, -12.5, [3, 9])
    g = m.gaussiansDF.toPandas()
    assert list(g.columns) == ["mean", "cov"] and len(g) == 2
    np.testing.assert_array_equal(np.stack(g["cov"][0]), [[1.0, 0.1], [0.1, 2.0]])
    assert m._transform_outputs() == [("prediction", "int"), ("prob", "array<double>")]
    for f in (lambda: m.predict([0.0, 0.0]), lambda: m.predictProbability([0.0, 0.0]), m.cpu):
        with pytest.raises(NotImplementedError):
            f()
    m.write().overwrite().save(str(tmp_path / "model"))
    m2 = GaussianMixtureModel.load(str(tmp_path / "model"))
    assert m2.weights_ == m.weights_ and m2.means_ == m.means_ and m2.covs_ == m.covs_
    assert m2.summary.clusterSizes == [3, 9] and m2.summary.logLikelihood == -12.5
    assert m2.getProbabilityCol() == "prob"
    est = GaussianMixture(k=3, tol=0.2)
    est.save(str(tmp_path / "est"))
    e2 = GaussianMixture.load(str(tmp_path / "est"))
    assert e2.getK() == 3 and e2.getTol() == 0.2 and e2.cuml_params["n_components"] == 3
