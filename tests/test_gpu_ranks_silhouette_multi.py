"""b2k_silhouette_multi at R = 2 and 3 ranks on one GPU through the in-process NCCL stand-in (child:
tests/_ranks_child_silhouette_multi.py): uneven shards, a rank with no rows, a cluster on the last rank only.  Every
rank gets the same bits, equal to each model's b2k_silhouette at the same R and within beta of the oracle; an error
raised by one rank's data fails on every rank with one message that names the model."""
import os
import pickle
import subprocess
import sys
import tempfile

import numpy as np
import pytest

import _ranks_child as child
import _ranks_child_silhouette_multi as multi_child
import silhouette_oracle as so

pytestmark = pytest.mark.gpu

CHILD = os.path.join(child.HERE, "_ranks_child_silhouette_multi.py")
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
            p = subprocess.run([sys.executable, CHILD, "silhouette_multi", str(R), out], env=env, cwd=child.ROOT,
                               capture_output=True, text=True, timeout=600)
            if p.returncode != 0 or not os.path.exists(out):
                pytest.fail(f"R={R}: the child failed (exit {p.returncode})\n{p.stdout[-2000:]}\n{p.stderr[-4000:]}")
            with open(out, "rb") as f:
                _RUNS[R] = pickle.load(f)
    return _RUNS[R]


@pytest.mark.parametrize("R", [2, 3])
@pytest.mark.parametrize("name,d,Ks,metric,path", multi_child.CASES)
def test_bits_equal_single_calls_on_every_rank(R, name, d, Ks, metric, path):
    c = _run(R)[name]
    assert "harness_error" not in c, c.get("harness_error")
    assert c["errs"] == [None] * R, c["errs"]
    assert c["group_error"] == "", c["group_error"]
    bits = [[np.float64(v).tobytes() for v in o["multi"]] for o in c["outs"]]
    assert all(b == bits[0] for b in bits)
    assert bits[0] == [np.float64(v).tobytes() for v in c["outs"][0]["single"]]
    X, ids = multi_child.data(d, Ks, seed=d + len(Ks))
    for v, i in zip(c["outs"][0]["multi"], ids):
        ref, beta = so.closed_form(X, i, metric), so.beta(X, i, metric, nranks=R)
        assert abs(v - ref) <= beta, (v, ref, beta)


@pytest.mark.parametrize("R", [2, 3])
@pytest.mark.parametrize("name,msg", [("nonfinite", "model 0: b2k_silhouette: features contain NaN or infinity"),
                                      ("one_cluster", "model 1: Number of clusters must be greater than one.")])
def test_errors_fail_on_every_rank(R, name, msg):
    c = _run(R)[name]
    assert "harness_error" not in c, c.get("harness_error")
    errs = c["errs"]
    assert all(e is not None for e in errs) and all(e == errs[0] for e in errs), errs
    assert msg in errs[0], errs[0]
    assert c["secs"] < RENDEZVOUS_TIMEOUT_S / 2, c["secs"]
