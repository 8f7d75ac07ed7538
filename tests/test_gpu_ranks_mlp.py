"""b2k_mlp_eval / b2k_mlp_fit at R = 2 and 3 ranks on one GPU through the in-process NCCL stand-in (child:
tests/_ranks_child_mlp.py), uneven shards with a one-row rank: every rank ends a fit with the same bits, an evaluation
agrees with one rank within 1e-12 of F, and of |grad F| on the fp64 path (the wgmma path adds each 512-row unit of
its gradient sums in fp32 before the fp64 fold, and a shard boundary moves the units, so there the gradient agrees
within 1e-6 of |grad F|), and a bad label, a NaN or (with kernel_path=2) a misaligned X on one rank fails every rank."""
import os
import pickle
import subprocess
import sys
import tempfile

import numpy as np
import pytest

import _ranks_child as child
import _ranks_child_mlp as mlp_child

pytestmark = pytest.mark.gpu

CHILD = os.path.join(child.HERE, "_ranks_child_mlp.py")
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
            p = subprocess.run([sys.executable, CHILD, "mlp", str(R), out], env=env, cwd=child.ROOT,
                               capture_output=True, text=True, timeout=600)
            if p.returncode != 0 or not os.path.exists(out):
                pytest.fail(f"R={R}: the child failed (exit {p.returncode})\n{p.stdout[-2000:]}\n{p.stderr[-4000:]}")
            with open(out, "rb") as f:
                _RUNS[R] = pickle.load(f)
    return _RUNS[R]


@pytest.mark.parametrize("R", [2, 3])
@pytest.mark.parametrize("name,layers,n", mlp_child.MLP_CASES)
def test_ranks_agree_with_one_rank(R, name, layers, n):
    c = _run(R)[name]
    assert "harness_error" not in c, c.get("harness_error")
    assert c["errs"] == [None] * R, c["errs"]
    first = c["outs"][0]
    for o in c["outs"]:
        np.testing.assert_array_equal(o["fit"]["weights"], first["fit"]["weights"])
        np.testing.assert_array_equal(o["fit"]["objective_history"], first["fit"]["objective_history"])
        assert o["F"] == first["F"] and np.array_equal(o["g"], first["g"]) and o["nt"] == n
    one = c["single"]
    assert abs(first["F"] - one["F"]) <= 1e-12 * abs(one["F"])
    gtol = 1e-6 if name == "wg" else 1e-12
    assert np.abs(first["g"] - one["g"]).max() <= gtol * np.linalg.norm(one["g"])
    np.testing.assert_allclose(first["fit"]["weights"], one["fit"]["weights"], rtol=1e-4 if name == "wg" else 1e-8,
                               atol=1e-6 if name == "wg" else 1e-10)


@pytest.mark.parametrize("R", [2, 3])
@pytest.mark.parametrize("name,msg", [("bad_label", "labels must be in [0, 2)"), ("nan", "NaN or an infinity"),
                                      ("misaligned", "kernel_path=2 requested")])
def test_bad_input_on_one_rank_fails_every_rank(R, name, msg):
    c = _run(R)[name]
    assert "harness_error" not in c, c.get("harness_error")
    errs = c["errs"]
    assert all(e is not None and msg in e for e in errs), errs
    assert c["secs"] < RENDEZVOUS_TIMEOUT_S / 2, c["secs"]
