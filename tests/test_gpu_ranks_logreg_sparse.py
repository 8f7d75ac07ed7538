"""The sparse logistic fit's multi-rank path on one GPU: R = 2 and 3 ranks as threads of a child interpreter
(tests/_ranks_child_logreg_sparse.py) through the in-process NCCL stand-in, with uneven shards and a rank whose rows are
all empty.  Every rank's model must be bitwise identical and close to the one-rank fit; an empty partition must fail on
every rank."""
import os
import pickle
import subprocess
import sys
import tempfile

import numpy as np
import pytest

import _ranks_child as rc
import _ranks_child_logreg_sparse as child

pytestmark = pytest.mark.gpu

CHILD = os.path.join(child.HERE, "_ranks_child_logreg_sparse.py")
RENDEZVOUS_TIMEOUT_S = 20
_RUNS = {}


def _run(R):
    if R not in _RUNS:
        env = dict(os.environ, B2K_NCCL_LIB=rc.FAKE_NCCL, B2K_FAKE_NCCL_TIMEOUT_S=str(RENDEZVOUS_TIMEOUT_S))
        if sys.flags.no_user_site:
            env["PYTHONNOUSERSITE"] = "1"
        with tempfile.TemporaryDirectory() as td:
            out = os.path.join(td, "out.pkl")
            p = subprocess.run([sys.executable, CHILD, str(R), out], env=env, cwd=rc.ROOT, capture_output=True,
                               text=True, timeout=600)
            if p.returncode != 0 or not os.path.exists(out):
                pytest.fail(f"R={R}: the child failed (exit {p.returncode})\n{p.stdout[-2000:]}\n{p.stderr[-4000:]}")
            with open(out, "rb") as f:
                _RUNS[R] = pickle.load(f)
    return _RUNS[R]


@pytest.mark.parametrize("R", [2, 3])
@pytest.mark.parametrize("name", ["binomial", "multinomial"])
def test_ranks_bitwise_identical_and_close_to_one_rank(R, name):
    c = _run(R)[name]
    assert "harness_error" not in c, c.get("harness_error")
    assert c["errs"] == [None] * R, c["errs"]
    bits = [o["bits"] for o in c["outs"]]
    assert all(b == bits[0] for b in bits)
    one = c["single"]
    np.testing.assert_allclose(c["outs"][0]["coef"], one["coef"], atol=1e-7)
    np.testing.assert_allclose(c["outs"][0]["icpt"], one["icpt"], atol=1e-7)


@pytest.mark.parametrize("R", [2, 3])
def test_empty_partition_fails_on_every_rank(R):
    c = _run(R)["fail_empty_rank"]
    assert "harness_error" not in c, c.get("harness_error")
    errs = c["errs"]
    assert all(e is not None and "empty partition" in e for e in errs), errs
    assert c["secs"] < RENDEZVOUS_TIMEOUT_S / 2, c["secs"]
