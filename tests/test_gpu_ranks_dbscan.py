"""DBSCAN's multi-rank path on one GPU: R = 2 and 3 ranks as threads of a child interpreter (tests/_ranks_child_dbscan.py)
through the in-process NCCL stand-in, with uneven shards, an empty rank and a rank smaller than one tile.  The labels,
core flags and cluster count of the ranks, put together in rank order, must equal the one-rank result bit for bit (and
the fp64 oracle); every error must reach every rank with the same message.  A two-GPU case over real NCCL follows
tests/test_gpu_multi.py and skips on one GPU."""
import os
import pickle
import subprocess
import sys
import tempfile

import numpy as np
import pytest

import _ranks_child as rc
import _ranks_child_dbscan as child
import dbscan_oracle as do

pytestmark = pytest.mark.gpu

CHILD = os.path.join(child.HERE, "_ranks_child_dbscan.py")
CHILD_TIMEOUT_S = 600
RENDEZVOUS_TIMEOUT_S = 20
RANKS = [2, 3]
_RUNS = {}
SPECS = {s[0]: s for s in child.case_specs()}


def _run(R):
    if R not in _RUNS:
        _RUNS[R] = _spawn(R)
    res = _RUNS[R]
    if isinstance(res, str):
        pytest.fail(res)
    return res


def _spawn(R):
    if not os.path.exists(rc.FAKE_NCCL):
        return f"{rc.FAKE_NCCL} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'`"
    env = dict(os.environ, B2K_NCCL_LIB=rc.FAKE_NCCL, B2K_FAKE_NCCL_TIMEOUT_S=str(RENDEZVOUS_TIMEOUT_S))
    if sys.flags.no_user_site:
        env["PYTHONNOUSERSITE"] = "1"
    with tempfile.TemporaryDirectory() as td:
        out = os.path.join(td, "out.pkl")
        try:
            p = subprocess.run([sys.executable, CHILD, str(R), out], env=env, cwd=rc.ROOT, capture_output=True,
                               text=True, timeout=CHILD_TIMEOUT_S)
        except subprocess.TimeoutExpired as e:
            return f"R={R}: the child timed out after {CHILD_TIMEOUT_S} s\n{(e.stderr or '')[-4000:]}"
        if p.returncode != 0 or not os.path.exists(out):
            return f"R={R}: the child failed (exit {p.returncode})\n{p.stdout[-2000:]}\n{p.stderr[-4000:]}"
        with open(out, "rb") as f:
            return pickle.load(f)


@pytest.mark.parametrize("R", RANKS)
@pytest.mark.parametrize("name", list(SPECS))
def test_ranks_equal_one_rank_bitwise(R, name):
    c = _run(R)[name]
    assert "harness_error" not in c, c.get("harness_error")
    assert c["errs"] == [None] * R, c["errs"]
    assert c["group_error"] == "", c["group_error"]
    assert c["trace"][0] and all(t == c["trace"][0] for t in c["trace"]), c["trace"]
    outs, one = c["outs"], c["single"]
    assert len({o["n_clusters"] for o in outs}) == 1
    assert len({o["path"] for o in outs}) == 1 and outs[0]["path"] == one["path"]
    lab = np.concatenate([o["labels"] for o in outs])
    core = np.concatenate([o["core"] for o in outs])
    sz = SPECS[name][6](len(one["labels"]), R)
    assert [len(o["labels"]) for o in outs] == sz
    np.testing.assert_array_equal(lab, one["labels"])
    np.testing.assert_array_equal(core, one["core"])
    assert outs[0]["n_clusters"] == one["n_clusters"]
    _, X, eps, ms, metric, _, _ = SPECS[name]
    ref = do.dbscan(X, float(eps), ms, metric)
    np.testing.assert_array_equal(lab, ref[0])
    np.testing.assert_array_equal(core, ref[1])
    assert one["n_clusters"] == ref[2] and ref[2] >= 1


@pytest.mark.parametrize("R", RANKS)
@pytest.mark.parametrize("name, msg", [("fail_nan", "DBSCAN input contains NaN or infinity"),
                                       ("fail_zero_row_cosine", "zero row"),
                                       ("fail_bad_eps", "eps = "),
                                       ("fail_bad_min_samples", "min_samples = 0"),
                                       ("fail_d_differs", "d differs between ranks")])
def test_every_rank_fails_together(R, name, msg):
    c = _run(R)[name]
    assert "harness_error" not in c, c.get("harness_error")
    errs = c["errs"]
    assert all(e is not None for e in errs), errs
    assert all(e == errs[0] for e in errs), errs
    assert msg in errs[0], errs[0]
    assert "timed out" not in c["group_error"], c["group_error"]
    assert c["secs"] < RENDEZVOUS_TIMEOUT_S / 2, c["secs"]


def _ngpu():
    import torch

    return torch.cuda.device_count()


@pytest.mark.skipif(_ngpu() < 2, reason="needs 2 GPUs")
def test_two_gpu_transform_matches_one_gpu():
    from spark_rapids_ml_b200.clustering import DBSCAN
    from spark_rapids_ml_b200.sparkshim import LocalSession

    X = child.blobs(20000, 16, 8, seed=7)
    out = []
    for w in (2, 1):
        s = LocalSession({"spark.rapids.ml.num_workers.local": str(w)})
        df = s.from_numpy(X, num_partitions=2)
        model = DBSCAN(eps=0.85 * np.sqrt(32), min_samples=5, num_workers=w).fit(df)
        out.append(np.array([r["prediction"] for r in model.transform(df).collect()]))
    np.testing.assert_array_equal(out[0], out[1])
    np.testing.assert_array_equal(out[0], do.dbscan(X, 0.85 * np.sqrt(32), 5)[0])
