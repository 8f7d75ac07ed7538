"""Logistic regression over two GPUs (skipped on a 1-GPU box): two barrier-task processes, the label pass's allgather,
the column-moments allreduces and one allreduce per evaluation.  Every rank runs the optimiser on the same allreduced
values, so both ranks must return bitwise-equal models; those must agree with the one-GPU fit of the same rows."""
import json
import os

import numpy as np
import pytest

import logreg_oracle as lo

pytestmark = pytest.mark.gpu


def _ngpu():
    import torch

    return torch.cuda.device_count()


def _fit_recording_ranks(est, df, out_dir):
    """Fits with every rank writing the model rows it computed to out_dir/rank<i>.json (only rank 0's reach the driver)."""
    orig = est._get_cuml_fit_func

    def recording(dataset, extra_params=None):
        fit = orig(dataset, extra_params)

        def wrapped(inputs, params):
            from spark_rapids_ml_b200.sparkshim import BarrierTaskContext

            res = fit(inputs, params)
            with open(os.path.join(out_dir, f"rank{BarrierTaskContext.get().partitionId()}.json"), "w") as f:
                json.dump(res, f)
            return res

        return wrapped

    est._get_cuml_fit_func = recording
    return est.fit(df)


@pytest.mark.skipif(_ngpu() < 2, reason="needs 2 GPUs")
@pytest.mark.parametrize("K,reg,a", [(2, 0.01, 0.0), (4, 0.02, 0.5)])
def test_two_rank_fit_is_rank_identical_and_matches_one_rank(tmp_path, K, reg, a):
    from spark_rapids_ml_b200.classification import LogisticRegression
    from spark_rapids_ml_b200.sparkshim import LocalSession

    rng = np.random.default_rng(K)
    n, d = 20000, 24
    X = (rng.normal(size=(n, d)) * (1 + np.arange(d) % 3) + 5.0).astype(np.float32)
    W = rng.normal(size=(K, d)) / np.sqrt(d)
    y = ((X.astype(np.float64) - 5.0) @ W.T + rng.gumbel(size=(n, K))).argmax(1).astype(np.float32)
    s = LocalSession({"spark.rapids.ml.num_workers.local": "2"})
    df = s.createDataFrame([(X[i].tolist(), float(y[i])) for i in range(n)], "features array<float>, label float",
                           num_partitions=2)
    params = dict(regParam=reg, elasticNetParam=a, tol=1e-12, maxIter=1000)
    m2 = _fit_recording_ranks(LogisticRegression(num_workers=2, **params), df, str(tmp_path))
    r0 = json.load(open(tmp_path / "rank0.json"))
    r1 = json.load(open(tmp_path / "rank1.json"))
    assert r0 == r1, "the two ranks returned different models"
    m1 = LogisticRegression(num_workers=1, **params).fit(df)
    W2, W1 = np.asarray(m2.coef_), np.asarray(m1.coef_)
    b2, b1 = np.asarray(m2.intercept_), np.asarray(m1.intercept_)
    # the ranks' partial sums are added in another order than one rank's: gradients differ by fp64 round-off only
    # (tests/logreg_oracle.py eval_bound), so both fits stop at the same optimum to the optimiser's tolerance
    assert np.abs(W2 - W1).max() <= 1e-6 * max(1.0, np.abs(W1).max())
    assert np.abs(b2 - b1).max() <= 1e-6 * max(1.0, np.abs(b1).max())
    P = lo.Problem(X, y, reg, a)
    theta = np.concatenate([(W2 * P.sig).ravel(), b2])
    assert P.residual(theta) <= 1e-8
