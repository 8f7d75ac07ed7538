"""b2k_bkm_fit at R = 2 and 3 ranks on one GPU through the in-process NCCL stand-in (child: tests/_ranks_child_bkm.py):
the tree has the one-rank structure and sizes, its values agree within fp64 tolerance, every rank returns the same
bits; an empty partition fails on every rank with one message."""
import os
import pickle
import subprocess
import sys
import tempfile

import numpy as np
import pytest

import _ranks_child as child
import _ranks_child_bkm as bkm_child

pytestmark = pytest.mark.gpu

CHILD = os.path.join(child.HERE, "_ranks_child_bkm.py")
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
            p = subprocess.run([sys.executable, CHILD, "bkm", str(R), out], env=env, cwd=child.ROOT,
                               capture_output=True, text=True, timeout=600)
            if p.returncode != 0 or not os.path.exists(out):
                pytest.fail(f"R={R}: the child failed (exit {p.returncode})\n{p.stdout[-2000:]}\n{p.stderr[-4000:]}")
            with open(out, "rb") as f:
                _RUNS[R] = pickle.load(f)
    return _RUNS[R]


@pytest.mark.parametrize("R", [2, 3])
@pytest.mark.parametrize("name,d,k,md", bkm_child.BKM_CASES)
def test_same_tree_as_one_rank(R, name, d, k, md):
    c = _run(R)[name]
    assert "harness_error" not in c, c.get("harness_error")
    assert c["errs"] == [None] * R, c["errs"]
    first = c["outs"][0]["fit"]
    for o in c["outs"]:
        for key in ("node_index", "centers", "sizes", "costs", "cluster_sizes"):
            np.testing.assert_array_equal(o["fit"][key], first[key])
        assert o["fit"]["training_cost"] == first["training_cost"]
    one = c["single"]["fit"]
    np.testing.assert_array_equal(first["node_index"], one["node_index"])
    np.testing.assert_array_equal(first["sizes"], one["sizes"])
    np.testing.assert_array_equal(first["cluster_sizes"], one["cluster_sizes"])
    np.testing.assert_allclose(first["centers"], one["centers"], rtol=0, atol=1e-11)
    np.testing.assert_allclose(first["costs"], one["costs"], rtol=1e-10, atol=1e-10)
    assert first["cluster_sizes"].sum() == 3000


@pytest.mark.parametrize("R", [2, 3])
def test_empty_partition_fails_on_every_rank(R):
    c = _run(R)["empty"]
    assert "harness_error" not in c, c.get("harness_error")
    errs = c["errs"]
    assert all(e is not None for e in errs) and all(e == errs[0] for e in errs), errs
    assert "empty partition (rank 1" in errs[0], errs[0]
    assert c["secs"] < RENDEZVOUS_TIMEOUT_S / 2, c["secs"]
