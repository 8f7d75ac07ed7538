"""The silhouette at R = 2 and 3 ranks on one GPU through the in-process NCCL stand-in (child:
tests/_ranks_child_silhouette.py): uneven shards, a rank with no rows, a cluster present on the last rank only.  Every
rank gets the same value, within the bound beta of the oracle and of the one-rank value; errors raised by one rank's
data fail on every rank with one message."""
import os
import pickle
import subprocess
import sys
import tempfile

import pytest

import _ranks_child as child
import _ranks_child_silhouette as sil_child
import silhouette_oracle as so

pytestmark = pytest.mark.gpu

CHILD = os.path.join(child.HERE, "_ranks_child_silhouette.py")
RENDEZVOUS_TIMEOUT_S = 20
_RUNS = {}


def _run(R):
    if R not in _RUNS:
        if not os.path.exists(child.FAKE_NCCL):
            pytest.fail(f"{child.FAKE_NCCL} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'`")
        env = dict(os.environ, B2K_NCCL_LIB=child.FAKE_NCCL, B2K_FAKE_NCCL_TIMEOUT_S=str(RENDEZVOUS_TIMEOUT_S))
        if sys.flags.no_user_site:
            env["PYTHONNOUSERSITE"] = "1"
        with tempfile.TemporaryDirectory() as td:
            out = os.path.join(td, "out.pkl")
            p = subprocess.run([sys.executable, CHILD, "silhouette", str(R), out], env=env, cwd=child.ROOT,
                               capture_output=True, text=True, timeout=600)
            if p.returncode != 0 or not os.path.exists(out):
                pytest.fail(f"R={R}: the child failed (exit {p.returncode})\n{p.stdout[-2000:]}\n{p.stderr[-4000:]}")
            with open(out, "rb") as f:
                _RUNS[R] = pickle.load(f)
    return _RUNS[R]


@pytest.mark.parametrize("R", [2, 3])
@pytest.mark.parametrize("name,d,K,metric,path", sil_child.SIL_CASES)
def test_value_identical_on_every_rank_and_within_beta(R, name, d, K, metric, path):
    c = _run(R)[name]
    assert "harness_error" not in c, c.get("harness_error")
    assert c["errs"] == [None] * R, c["errs"]
    assert c["group_error"] == "", c["group_error"]
    vals = [o["value"] for o in c["outs"]]
    assert all(v == vals[0] for v in vals), vals
    X, ids = sil_child.data(d, K, seed=d + K)
    ref, beta = so.closed_form(X, ids, metric), so.beta(X, ids, metric, nranks=R)
    assert abs(vals[0] - ref) <= beta, (vals[0], ref, beta)
    assert abs(vals[0] - c["single"]["value"]) <= 2 * beta, (vals[0], c["single"]["value"], beta)


@pytest.mark.parametrize("R", [2, 3])
@pytest.mark.parametrize("name,msg", [("nonfinite", "NaN or infinity"),
                                      ("one_cluster", "Number of clusters must be greater than one.")])
def test_errors_fail_on_every_rank(R, name, msg):
    c = _run(R)[name]
    assert "harness_error" not in c, c.get("harness_error")
    errs = c["errs"]
    assert all(e is not None for e in errs) and all(e == errs[0] for e in errs), errs
    assert msg in errs[0], errs[0]
    assert c["secs"] < RENDEZVOUS_TIMEOUT_S / 2, c["secs"]
