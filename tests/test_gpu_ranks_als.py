"""b2k_als_fit at R = 2 and 3 ranks on one GPU through the in-process NCCL stand-in (child: tests/_ranks_child_als.py),
uneven shards with a rank that holds no ratings and users whose ratings span ranks: every rank returns the one-rank
factors and id maps bit for bit (explicit and implicit), and a bad id or a NaN rating on one rank fails every rank."""
import os
import pickle
import subprocess
import sys
import tempfile

import numpy as np
import pytest

import _ranks_child as child
import _ranks_child_als as als_child

pytestmark = pytest.mark.gpu

CHILD = os.path.join(child.HERE, "_ranks_child_als.py")
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
            p = subprocess.run([sys.executable, CHILD, "als", str(R), out], env=env, cwd=child.ROOT,
                               capture_output=True, text=True, timeout=600)
            if p.returncode != 0 or not os.path.exists(out):
                pytest.fail(f"R={R}: the child failed (exit {p.returncode})\n{p.stdout[-2000:]}\n{p.stderr[-4000:]}")
            with open(out, "rb") as f:
                _RUNS[R] = pickle.load(f)
    return _RUNS[R]


@pytest.mark.parametrize("R", [2, 3])
@pytest.mark.parametrize("name,rank,implicit", als_child.ALS_CASES)
def test_ranks_equal_one_rank_bitwise(R, name, rank, implicit):
    c = _run(R)[name]
    assert "harness_error" not in c, c.get("harness_error")
    assert c["errs"] == [None] * R, c["errs"]
    u = als_child.data(rank, implicit)[0]
    sz = als_child.shard_sizes(R)
    # some user's ratings sit on two ranks
    assert len(np.intersect1d(u[:sz[0]], u[sz[0]:])) > 0
    one = c["single"]
    for o in c["outs"]:
        for k in ("user_ids", "item_ids", "user_factors", "item_factors"):
            np.testing.assert_array_equal(o[k], one[k])


@pytest.mark.parametrize("R", [2, 3])
@pytest.mark.parametrize("name,msg", [("bad_id", "Integer range"), ("nan", "finite ratings")])
def test_bad_input_on_one_rank_fails_every_rank(R, name, msg):
    c = _run(R)[name]
    assert "harness_error" not in c, c.get("harness_error")
    errs = c["errs"]
    assert all(e is not None and msg in e for e in errs), errs
    assert c["secs"] < RENDEZVOUS_TIMEOUT_S / 2, c["secs"]
